// Non-GEMM kernels of the DINO ViT forward: pixel normalisation + im2col, CLS row, LayerNorm, CLS attention row.
#include <math.h>

#include "common.cuh"

namespace dss {

// ---------------------------------------------------------------------------------------------------------------
// im2col: images_u8 [B,H,W,3] -> patches f16 [B*Np, 3*P*P]; column = c*P*P + py*P + px (the flattening of the
// Conv2d weight [d,3,P,P]); value = ((u8/255) - mean_c)/std_c  (ToTensor + Normalize, extract_utils.py:53-59).
// The crop to patch multiples (extract.py:82-88) is implicit: only pixels of whole patches are read.
__constant__ float c_mean[3] = {0.485f, 0.456f, 0.406f};
__constant__ float c_std[3] = {0.229f, 0.224f, 0.225f};

// One thread = 8 consecutive pixels of one patch row, ALL three channels: it reads the 24 interleaved RGB bytes once
// (32-bit loads when the address allows; consecutive threads read consecutive 24-byte spans, so a warp covers one
// contiguous stretch of the image row) and writes three 16-byte stores, one per channel plane of the patch.
// (Round 1 used one thread per channel with byte loads at stride 3: every input byte was fetched three times; 0.19 of
// the HBM roofline.)
__global__ void im2col_f16_kernel(const uint8_t* __restrict__ img, __half* __restrict__ out, int B, int H, int W, int P,
                                  int Hp, int Wp) {
  const int groups_per_row = P / 8;                       // 8-px groups per patch row
  const int per_patch = P * groups_per_row;               // (py, group) pairs per patch
  const long long total = (long long)B * Hp * Wp * per_patch;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  // consecutive threads walk along an image row: (b, patch row ph, py, patch column pw, group)
  const int g = (int)(gid % groups_per_row);
  const int pw = (int)((gid / groups_per_row) % Wp);
  const int py = (int)((gid / ((long long)groups_per_row * Wp)) % P);
  const int ph = (int)((gid / ((long long)groups_per_row * Wp * P)) % Hp);
  const int b = (int)(gid / ((long long)groups_per_row * Wp * P * Hp));
  const int px0 = g * 8;
  const uint8_t* src = img + (((long long)b * H + (ph * P + py)) * W + (pw * P + px0)) * 3;
  uint8_t raw[24];
  if ((reinterpret_cast<uintptr_t>(src) & 3) == 0) {
    const uint32_t* s4 = reinterpret_cast<const uint32_t*>(src);
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      const uint32_t w = __ldg(s4 + i);
      raw[4 * i] = w & 0xff; raw[4 * i + 1] = (w >> 8) & 0xff; raw[4 * i + 2] = (w >> 16) & 0xff; raw[4 * i + 3] = w >> 24;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 24; ++i) raw[i] = __ldg(src + i);
  }
  const long long patch = ((long long)b * Hp + ph) * Wp + pw;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float mean = c_mean[c], sd = c_std[c];
    float v[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) v[t] = (static_cast<float>(raw[t * 3 + c]) / 255.0f - mean) / sd;
    uint4 q;
    q.x = pack_half2(v[0], v[1]);
    q.y = pack_half2(v[2], v[3]);
    q.z = pack_half2(v[4], v[5]);
    q.w = pack_half2(v[6], v[7]);
    __half* dst = out + patch * (3LL * P * P) + (c * P + py) * P + px0;
    *reinterpret_cast<uint4*>(dst) = q;
  }
}

// x[b, 0, :] = cls + pos[0, :]
__global__ void cls_row_kernel(float* __restrict__ x, const float* __restrict__ cls, const float* __restrict__ pos,
                               int B, int T, int d) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * d) return;
  const int b = i / d, c = i % d;
  x[(long long)b * T * d + c] = cls[c] + pos[c];
}

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, row kept in registers, two-pass variance (mean, then E[(x-mean)^2]) like torch,
// in the explicitly rounded arithmetic of the ln_* helpers (common.cuh).
template <int D>
__global__ void __launch_bounds__(256)
layernorm_f16_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                     __half* __restrict__ y, int M, float eps) {
  constexpr int V = D / 128;  // float4 per lane
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
  uint2* yr = reinterpret_cast<uint2*>(y + (long long)warp * D);
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32 * i);
    const float4 bt = __ldg(reinterpret_cast<const float4*>(beta) + lane + 32 * i);
    const uint2 o = ln_out4(v[i], rstd, g, bt);
    yr[lane + 32 * i] = o;
  }
}

// ---------------------------------------------------------------------------------------------------------------
int launch_im2col(const uint8_t* img, void* patches, int B, int H, int W, int P, cudaStream_t st) {
  DSS_REQUIRE(P % 8 == 0 && P > 0, "im2col: patch must be a multiple of 8 (got %d)", P);
  const int Hp = H / P, Wp = W / P;
  DSS_REQUIRE(B > 0 && Hp > 0 && Wp > 0, "im2col: image %dx%d smaller than one patch", H, W);
  const long long total = (long long)B * Hp * Wp * P * (P / 8);
  const int threads = 256;
  LaunchScope scope(st, KC_IM2COL);
  im2col_f16_kernel<<<(unsigned)((total + threads - 1) / threads), threads, 0, st>>>(
      img, reinterpret_cast<__half*>(patches), B, H, W, P, Hp, Wp);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

// Zero-padded variant (object-localization/main.py:227-235 pads the normalised image with zeros up to multiples of
// P): the grid is ceil(H/P) x ceil(W/P); a pixel outside the image is 0. One thread = 8 pixels of one patch row.
__global__ void im2col_pad_f16_kernel(const uint8_t* __restrict__ img, __half* __restrict__ out, int B, int H, int W,
                                      int P, int Hp, int Wp) {
  const int groups_per_row = P / 8;
  const long long total = (long long)B * Hp * Wp * P * groups_per_row;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  const int g = (int)(gid % groups_per_row);
  const int pw = (int)((gid / groups_per_row) % Wp);
  const int py = (int)((gid / ((long long)groups_per_row * Wp)) % P);
  const int ph = (int)((gid / ((long long)groups_per_row * Wp * P)) % Hp);
  const int b = (int)(gid / ((long long)groups_per_row * Wp * P * Hp));
  const int y = ph * P + py, x0 = pw * P + g * 8;
  const long long patch = ((long long)b * Hp + ph) * Wp + pw;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float mean = c_mean[c], sd = c_std[c];
    float v[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int x = x0 + t;
      v[t] = (y < H && x < W) ? (static_cast<float>(__ldg(img + (((long long)b * H + y) * W + x) * 3 + c)) / 255.0f - mean) / sd
                              : 0.f;
    }
    uint4 q;
    q.x = pack_half2(v[0], v[1]);
    q.y = pack_half2(v[2], v[3]);
    q.z = pack_half2(v[4], v[5]);
    q.w = pack_half2(v[6], v[7]);
    *reinterpret_cast<uint4*>(out + patch * (3LL * P * P) + (c * P + py) * P + g * 8) = q;
  }
}

int launch_im2col_pad(const uint8_t* img, void* patches, int B, int H, int W, int P, cudaStream_t st) {
  DSS_REQUIRE(P % 8 == 0 && P > 0, "im2col_pad: patch must be a multiple of 8 (got %d)", P);
  DSS_REQUIRE(B > 0 && H > 0 && W > 0, "im2col_pad: empty image batch");
  const int Hp = cdiv(H, P), Wp = cdiv(W, P);
  const long long total = (long long)B * Hp * Wp * P * (P / 8);
  const int threads = 256;
  LaunchScope scope(st, KC_IM2COL);
  im2col_pad_f16_kernel<<<(unsigned)((total + threads - 1) / threads), threads, 0, st>>>(
      img, reinterpret_cast<__half*>(patches), B, H, W, P, Hp, Wp);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

// CLS row of the last block's attention (get_last_selfattention(...)[:, :, 0, 1:], the input of dino_seg):
// s_j = (q_0 . k_j) / 8 over all T tokens, softmax in fp32. One CTA per (head, image); the 64-term dot products are
// recomputed in each of the three passes (max, sum, output) rather than kept in scratch memory.
constexpr int CLSATT_THREADS = 256;
__device__ __forceinline__ float cls_score(const float* q0, const __half* k) {
  float acc = 0.f;
#pragma unroll 8
  for (int i = 0; i < 64; ++i) acc = fmaf(q0[i], __half2float(k[i]), acc);
  return acc * 0.125f;
}
__device__ __forceinline__ float cls_block_reduce(float v, float* red, bool is_max) {
  v = is_max ? warp_max(v) : warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < CLSATT_THREADS / 32 ? red[threadIdx.x] : (is_max ? -INFINITY : 0.f);
    t = is_max ? warp_max(t) : warp_sum(t);
    if (threadIdx.x == 0) red[CLSATT_THREADS / 32] = t;
  }
  __syncthreads();
  return red[CLSATT_THREADS / 32];
}
__global__ void __launch_bounds__(CLSATT_THREADS)
cls_attention_kernel(const __half* __restrict__ qkv, int T, int heads, float* __restrict__ out) {
  __shared__ float q0[64];
  __shared__ float red[CLSATT_THREADS / 32 + 1];
  const int h = blockIdx.x, b = blockIdx.y, d = heads * 64, tid = threadIdx.x;
  const __half* base = qkv + (long long)b * T * 3 * d;
  const __half* kbase = base + d + h * 64;
  if (tid < 64) q0[tid] = __half2float(base[h * 64 + tid]);
  __syncthreads();
  float mx = -INFINITY;
  for (int j = tid; j < T; j += CLSATT_THREADS) mx = fmaxf(mx, cls_score(q0, kbase + (long long)j * 3 * d));
  mx = cls_block_reduce(mx, red, true);
  float sum = 0.f;
  for (int j = tid; j < T; j += CLSATT_THREADS) sum += expf(cls_score(q0, kbase + (long long)j * 3 * d) - mx);
  sum = cls_block_reduce(sum, red, false);
  float* o = out + ((long long)b * heads + h) * (T - 1);
  for (int j = tid + 1; j < T; j += CLSATT_THREADS) o[j - 1] = expf(cls_score(q0, kbase + (long long)j * 3 * d) - mx) / sum;
}

int launch_cls_attention(const void* qkv, int B, int T, int heads, float* out, cudaStream_t st) {
  DSS_REQUIRE(B > 0 && T >= 2 && heads > 0, "cls_attention: bad shape (B=%d T=%d heads=%d)", B, T, heads);
  LaunchScope scope(st, KC_ATTENTION);
  cls_attention_kernel<<<dim3(heads, B), CLSATT_THREADS, 0, st>>>(reinterpret_cast<const __half*>(qkv), T, heads, out);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_cls_row(float* x, const float* cls, const float* pos, int B, int T, int d, cudaStream_t st) {
  LaunchScope scope(st, KC_CLS_ROW);
  cls_row_kernel<<<cdiv(B * d, 256), 256, 0, st>>>(x, cls, pos, B, T, d);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_layernorm(const float* x, const float* g, const float* b, void* y, int M, int d, float eps,
                     cudaStream_t st) {
  DSS_REQUIRE(d == 384 || d == 768, "layernorm: d must be 384 or 768 (got %d)", d);
  DSS_REQUIRE(M > 0, "layernorm: empty input");
  const int threads = 256;  // 8 rows per CTA
  const int grid = cdiv(M, threads / 32);
  LaunchScope scope(st, KC_LAYERNORM);
  if (d == 384)
    layernorm_f16_kernel<384><<<grid, threads, 0, st>>>(x, g, b, reinterpret_cast<__half*>(y), M, eps);
  else
    layernorm_f16_kernel<768><<<grid, threads, 0, st>>>(x, g, b, reinterpret_cast<__half*>(y), M, eps);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

}  // namespace dss

using namespace dss;

extern "C" int dss_op_layernorm_f16(const float* x, const float* gamma, const float* beta, void* y, int M, int d,
                                    float eps, dss_stream_t stream) {
  return launch_layernorm(x, gamma, beta, y, M, d, eps, static_cast<cudaStream_t>(stream));
}
extern "C" int dss_op_im2col_f16(const uint8_t* images_u8, void* patches, int B, int H, int W, int P,
                                 dss_stream_t stream) {
  return launch_im2col(images_u8, patches, B, H, W, P, static_cast<cudaStream_t>(stream));
}
extern "C" int dss_op_im2col_pad_f16(const uint8_t* images_u8, void* patches, int B, int H, int W, int P,
                                     dss_stream_t stream) {
  DSS_REQUIRE(images_u8 && patches, "im2col_pad: null pointer");
  return launch_im2col_pad(images_u8, patches, B, H, W, P, static_cast<cudaStream_t>(stream));
}
extern "C" int dss_op_cls_attention(const void* qkv, int B, int T, int heads, float* cls_attn, dss_stream_t stream) {
  DSS_REQUIRE(qkv && cls_attn, "cls_attention: null pointer");
  DSS_REQUIRE(B > 0 && T >= 2 && heads > 0, "cls_attention: bad shape (B=%d T=%d heads=%d)", B, T, heads);
  return launch_cls_attention(qkv, B, T, heads, cls_attn, static_cast<cudaStream_t>(stream));
}
