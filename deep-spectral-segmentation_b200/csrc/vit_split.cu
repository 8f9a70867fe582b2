// Split-fp16 operand producers of the fp32-precision ViT (DSS_VIT_PRECISION_FP32): every value that feeds a tensor-core
// product is written as the three fp16 groups of split_f16 (common.cuh), so that one fp16 GEMM over K' = 3 K gives the
// fp32-equivalent product. A operands (activations) are rows [hi | hi/64 | 64 lo], each group K wide; B operands
// (weights, and K / V of attention) are [hi | 64 lo | hi/64]. The fp32 value that is split is the one the fp16 path
// rounds (im2col, LayerNorm) or the fp32 output of the preceding GEMM (qkv, fc1 + exact-erf GELU).
#include <math.h>

#include "common.cuh"

namespace dss {

__constant__ float c_split_mean[3] = {0.485f, 0.456f, 0.406f};
__constant__ float c_split_std[3] = {0.229f, 0.224f, 0.225f};

// fp32 [rows, cols] -> split [rows, 3 cols], order 0 = A ([hi | hi/64 | 64 lo]), 1 = B ([hi | 64 lo | hi/64])
__global__ void split_rows_kernel(const float* __restrict__ x, __half* __restrict__ out, long long rows, int cols,
                                  int order) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const long long r = i / cols;
  const int c = (int)(i % cols);
  const SplitF16 s = split_f16(x[i]);
  __half* o = out + r * 3 * cols + c;
  o[0] = s.hi;
  o[cols] = order ? s.lo_s : s.hi_s;
  o[2 * cols] = order ? s.hi_s : s.lo_s;
}

// im2col of DSS_VIT_PRECISION_FP32: patches [B*Np, 3 * 3P^2] in A order. The value is im2col_f16_kernel's
// ((u8/255) - mean_c)/std_c; pixels outside the image (the zero-padded grid) are 0. One thread per patch element.
__global__ void im2col_split_kernel(const uint8_t* __restrict__ img, __half* __restrict__ out, int B, int H, int W,
                                    int P, int Hp, int Wp) {
  const int Kp = 3 * P * P;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * Hp * Wp * Kp) return;
  const long long patch = i / Kp;
  const int col = (int)(i % Kp), c = col / (P * P), py = (col / P) % P, px = col % P;
  const int pw = (int)(patch % Wp), ph = (int)((patch / Wp) % Hp), b = (int)(patch / ((long long)Wp * Hp));
  const int y = ph * P + py, x = pw * P + px;
  const float v = (y < H && x < W)
                      ? (static_cast<float>(img[(((long long)b * H + y) * W + x) * 3 + c]) / 255.0f - c_split_mean[c]) / c_split_std[c]
                      : 0.f;
  const SplitF16 s = split_f16(v);
  __half* o = out + patch * 3 * Kp + col;
  o[0] = s.hi;
  o[Kp] = s.hi_s;
  o[2 * Kp] = s.lo_s;
}

// LayerNorm with layernorm_f16_kernel's statistics and output arithmetic (the ln_* helpers), written in A order
// [M, 3D]. A sibling rather than a template of that kernel so the fp16 path's code is untouched.
template <int D>
__global__ void __launch_bounds__(256)
layernorm_split_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                       __half* __restrict__ y, int M, float eps) {
  constexpr int V = D / 128;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= M) return;
  const float4* xr = reinterpret_cast<const float4*>(x + (long long)warp * D);
  float4 v[V];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    v[i] = xr[lane + 32 * i];
    s = __fadd_rn(s, ln_sum4(v[i]));
  }
  const float S = warp_sum(s);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    v[i] = ln_center4(v[i], S, 1.0f / D);
    q = __fadd_rn(q, ln_sq4(v[i]));
  }
  const float rstd = ln_rstd(warp_sum(q), 1.0f / D, eps);
  __half* yr = y + (long long)warp * 3 * D;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32 * i);
    const float4 bt = __ldg(reinterpret_cast<const float4*>(beta) + lane + 32 * i);
    const float o[4] = {__fmaf_rn(__fmul_rn(v[i].x, rstd), g.x, bt.x), __fmaf_rn(__fmul_rn(v[i].y, rstd), g.y, bt.y),
                        __fmaf_rn(__fmul_rn(v[i].z, rstd), g.z, bt.z), __fmaf_rn(__fmul_rn(v[i].w, rstd), g.w, bt.w)};
    const int c = 4 * (lane + 32 * i);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const SplitF16 sp = split_f16(o[t]);
      yr[c + t] = sp.hi;
      yr[D + c + t] = sp.hi_s;
      yr[2 * D + c + t] = sp.lo_s;
    }
  }
}

// MLP hidden activations: h [M, n] fp32 (fc1 output, bias included) -> gelu(h) in A order [M, 3n]. Exact erf, as
// torch's GELU: the polynomial gelu_erf of the fp16 path is accurate to 6.4e-6 only, an fp16-level error.
__global__ void gelu_split_kernel(const float* __restrict__ h, __half* __restrict__ out, long long M, int n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * n) return;
  const float x = h[i];
  const SplitF16 s = split_f16(0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)));
  __half* o = out + (i / n) * 3 * n + (int)(i % n);
  o[0] = s.hi;
  o[n] = s.hi_s;
  o[2 * n] = s.lo_s;
}

// qkv [M, 3d] fp32 (qkv GEMM output) -> per-head attention operands [M, 9d]: Q'_h at columns h*192 in A order, K'_h at
// 3d + h*192 and V'_h at 6d + h*192 in B order ([hi | 64 lo | hi/64], 64 columns each).
__global__ void qkv_split_kernel(const float* __restrict__ qkv, __half* __restrict__ out, long long M, int d) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * 3 * d) return;
  const long long r = i / (3 * d);
  const int c = (int)(i % (3 * d)), which = c / d, head = (c % d) >> 6, j = c & 63;
  const SplitF16 s = split_f16(qkv[i]);
  __half* o = out + r * 9 * d + (long long)which * 3 * d + head * 192 + j;
  o[0] = s.hi;
  o[64] = which ? s.lo_s : s.hi_s;
  o[128] = which ? s.hi_s : s.lo_s;
}

// CLS attention row from the fp32 qkv of DSS_VIT_PRECISION_FP32 (cls_attention_kernel's arithmetic on fp32 keys)
constexpr int CLSF_THREADS = 256;
__device__ __forceinline__ float cls_score_f32(const float* q0, const float* k) {
  float acc = 0.f;
#pragma unroll 8
  for (int i = 0; i < 64; ++i) acc = fmaf(q0[i], k[i], acc);
  return acc * 0.125f;
}
__device__ __forceinline__ float clsf_block_reduce(float v, float* red, bool is_max) {
  v = is_max ? warp_max(v) : warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < CLSF_THREADS / 32 ? red[threadIdx.x] : (is_max ? -INFINITY : 0.f);
    t = is_max ? warp_max(t) : warp_sum(t);
    if (threadIdx.x == 0) red[CLSF_THREADS / 32] = t;
  }
  __syncthreads();
  return red[CLSF_THREADS / 32];
}
__global__ void __launch_bounds__(CLSF_THREADS)
cls_attention_f32_kernel(const float* __restrict__ qkv, int T, int heads, float* __restrict__ out) {
  __shared__ float q0[64];
  __shared__ float red[CLSF_THREADS / 32 + 1];
  const int h = blockIdx.x, b = blockIdx.y, d = heads * 64, tid = threadIdx.x;
  const float* base = qkv + (long long)b * T * 3 * d;
  const float* kbase = base + d + h * 64;
  if (tid < 64) q0[tid] = base[h * 64 + tid];
  __syncthreads();
  float mx = -INFINITY;
  for (int j = tid; j < T; j += CLSF_THREADS) mx = fmaxf(mx, cls_score_f32(q0, kbase + (long long)j * 3 * d));
  mx = clsf_block_reduce(mx, red, true);
  float sum = 0.f;
  for (int j = tid; j < T; j += CLSF_THREADS) sum += expf(cls_score_f32(q0, kbase + (long long)j * 3 * d) - mx);
  sum = clsf_block_reduce(sum, red, false);
  float* o = out + ((long long)b * heads + h) * (T - 1);
  for (int j = tid + 1; j < T; j += CLSF_THREADS)
    o[j - 1] = expf(cls_score_f32(q0, kbase + (long long)j * 3 * d) - mx) / sum;
}

static unsigned grid_for(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

int launch_split_rows(const float* x, void* out, long long rows, int cols, int order, cudaStream_t st, int kclass) {
  DSS_REQUIRE(x && out, "split: null pointer");
  DSS_REQUIRE(rows > 0 && cols > 0 && (order == 0 || order == 1), "split: bad arguments rows=%lld cols=%d order=%d",
              rows, cols, order);
  LaunchScope scope(st, kclass);
  split_rows_kernel<<<grid_for(rows * cols, 256), 256, 0, st>>>(x, reinterpret_cast<__half*>(out), rows, cols, order);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_im2col_split(const uint8_t* img, void* patches, int B, int H, int W, int P, int pad, cudaStream_t st) {
  DSS_REQUIRE(img && patches, "im2col_split: null pointer");
  DSS_REQUIRE(P > 0 && B > 0 && H > 0 && W > 0, "im2col_split: bad shape");
  const int Hp = pad ? cdiv(H, P) : H / P, Wp = pad ? cdiv(W, P) : W / P;
  DSS_REQUIRE(Hp > 0 && Wp > 0, "im2col_split: image %dx%d smaller than one patch", H, W);
  LaunchScope scope(st, KC_IM2COL);
  im2col_split_kernel<<<grid_for((long long)B * Hp * Wp * 3 * P * P, 256), 256, 0, st>>>(
      img, reinterpret_cast<__half*>(patches), B, H, W, P, Hp, Wp);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_layernorm_split(const float* x, const float* g, const float* b, void* y, int M, int d, float eps,
                           cudaStream_t st) {
  DSS_REQUIRE(d == 384 || d == 768, "layernorm_split: d must be 384 or 768 (got %d)", d);
  DSS_REQUIRE(M > 0, "layernorm_split: empty input");
  const int grid = cdiv(M, 8);
  LaunchScope scope(st, KC_LAYERNORM);
  if (d == 384)
    layernorm_split_kernel<384><<<grid, 256, 0, st>>>(x, g, b, reinterpret_cast<__half*>(y), M, eps);
  else
    layernorm_split_kernel<768><<<grid, 256, 0, st>>>(x, g, b, reinterpret_cast<__half*>(y), M, eps);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_gelu_split(const float* h, void* out, long long M, int n, cudaStream_t st) {
  DSS_REQUIRE(h && out && M > 0 && n > 0, "gelu_split: bad arguments");
  LaunchScope scope(st, KC_GEMM_FC1);
  gelu_split_kernel<<<grid_for(M * n, 256), 256, 0, st>>>(h, reinterpret_cast<__half*>(out), M, n);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_qkv_split(const float* qkv, void* out, long long M, int d, cudaStream_t st) {
  DSS_REQUIRE(qkv && out && M > 0 && d % 64 == 0, "qkv_split: bad arguments");
  LaunchScope scope(st, KC_ATTENTION);
  qkv_split_kernel<<<grid_for(M * 3 * d, 256), 256, 0, st>>>(qkv, reinterpret_cast<__half*>(out), M, d);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_cls_attention_f32(const float* qkv, int B, int T, int heads, float* out, cudaStream_t st) {
  DSS_REQUIRE(B > 0 && T >= 2 && heads > 0, "cls_attention: bad shape (B=%d T=%d heads=%d)", B, T, heads);
  LaunchScope scope(st, KC_ATTENTION);
  cls_attention_f32_kernel<<<dim3(heads, B), CLSF_THREADS, 0, st>>>(qkv, T, heads, out);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

}  // namespace dss

using namespace dss;

extern "C" int dss_op_split_f16(const float* x, void* out, int rows, int cols, int order, dss_stream_t stream) {
  return launch_split_rows(x, out, rows, cols, order, static_cast<cudaStream_t>(stream), KC_MISC);
}
extern "C" int dss_op_layernorm_split_f16(const float* x, const float* gamma, const float* beta, void* y, int M, int d,
                                          float eps, dss_stream_t stream) {
  DSS_REQUIRE(x && gamma && beta && y, "layernorm_split: null pointer");
  return launch_layernorm_split(x, gamma, beta, y, M, d, eps, static_cast<cudaStream_t>(stream));
}
extern "C" int dss_op_gelu_split_f16(const float* h, void* out, int M, int n, dss_stream_t stream) {
  return launch_gelu_split(h, out, M, n, static_cast<cudaStream_t>(stream));
}
extern "C" int dss_op_im2col_split_f16(const uint8_t* images_u8, void* patches, int B, int H, int W, int P, int pad,
                                       dss_stream_t stream) {
  return launch_im2col_split(images_u8, patches, B, H, W, P, pad, static_cast<cudaStream_t>(stream));
}
