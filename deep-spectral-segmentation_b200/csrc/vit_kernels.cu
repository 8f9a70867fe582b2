// Non-GEMM kernels of the DINO ViT forward: pixel normalisation + im2col, LayerNorm, CLS attention row, and
// the split-fp16 operand producers of DSS_VIT_PRECISION_FP32. In that mode every value that feeds a tensor-core
// product is written as the three fp16 groups of split_f16 (common.cuh), so that one fp16 GEMM over K' = 3 K gives the
// fp32-equivalent product: activations in A order, weights (and K / V of attention) in B order. The fp32 value that is
// split is the one the fp16 path rounds (im2col, LayerNorm) or the fp32 output of the preceding GEMM (qkv, fc1 +
// exact-erf GELU).
#include <math.h>

#include "common.cuh"

namespace dss {

static unsigned grid_for(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// ---------------------------------------------------------------------------------------------------------------
// im2col: images_u8 [B,H,W,3] -> patches [B*Np, 3*P*P]; column = c*P*P + py*P + px (the flattening of the Conv2d
// weight [d,3,P,P]); value = ((u8/255) - mean_c)/std_c  (ToTensor + Normalize, extract_utils.py:53-59).
// The crop to patch multiples (extract.py:82-88) is implicit: only pixels of whole patches are read. The zero-padded
// grid (object-localization/main.py:227-235 pads the normalised image with zeros up to multiples of P) is
// ceil(H/P) x ceil(W/P); a pixel outside the image is 0.
__constant__ float c_mean[3] = {0.485f, 0.456f, 0.406f};
__constant__ float c_std[3] = {0.229f, 0.224f, 0.225f};
__device__ __forceinline__ float pixel_value(uint8_t u8, int c) {
  return (static_cast<float>(u8) / 255.0f - c_mean[c]) / c_std[c];
}

// One thread = 8 consecutive pixels of one patch row, ALL three channels, written as three 16-byte stores, one per
// channel plane of the patch. The crop (PAD false) reads the 24 interleaved RGB bytes once (32-bit loads when the
// address allows; consecutive threads read consecutive 24-byte spans, so a warp covers one contiguous stretch of the
// image row); the padded grid reads bytes, each checked against the image bounds.
// (Round 1 used one thread per channel with byte loads at stride 3: every input byte was fetched three times; 0.19 of
// the HBM roofline.)
template <bool PAD>
__global__ void im2col_f16_kernel(const uint8_t* __restrict__ img, __half* __restrict__ out, int B, int H, int W, int P,
                                  int Hp, int Wp) {
  const int groups_per_row = P / 8;                       // 8-px groups per patch row
  const int per_patch = P * groups_per_row;               // (py, group) pairs per patch
  const long long total = PAD ? (long long)B * Hp * Wp * P * groups_per_row : (long long)B * Hp * Wp * per_patch;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  // consecutive threads walk along an image row: (b, patch row ph, py, patch column pw, group)
  const int g = (int)(gid % groups_per_row);
  const int pw = (int)((gid / groups_per_row) % Wp);
  const int py = (int)((gid / ((long long)groups_per_row * Wp)) % P);
  const int ph = (int)((gid / ((long long)groups_per_row * Wp * P)) % Hp);
  const int b = (int)(gid / ((long long)groups_per_row * Wp * P * Hp));
  const int px0 = g * 8;
  auto store = [&](int c, const float (&v)[8]) {
    const long long patch = ((long long)b * Hp + ph) * Wp + pw;
    uint4 q;
    q.x = pack_half2(v[0], v[1]);
    q.y = pack_half2(v[2], v[3]);
    q.z = pack_half2(v[4], v[5]);
    q.w = pack_half2(v[6], v[7]);
    *reinterpret_cast<uint4*>(out + patch * (3LL * P * P) + (c * P + py) * P + px0) = q;
  };
  if constexpr (PAD) {
    const int y = ph * P + py, x0 = pw * P + px0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v[8];
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const int x = x0 + t;
        v[t] = (y < H && x < W) ? pixel_value(__ldg(img + (((long long)b * H + y) * W + x) * 3 + c), c) : 0.f;
      }
      store(c, v);
    }
  } else {
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
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v[8];
#pragma unroll
      for (int t = 0; t < 8; ++t) v[t] = pixel_value(raw[t * 3 + c], c);
      store(c, v);
    }
  }
}

// im2col of DSS_VIT_PRECISION_FP32: patches [B*Np, 3 * 3P^2] in A order, crop or padded grid. One thread per patch
// element.
__global__ void im2col_split_kernel(const uint8_t* __restrict__ img, __half* __restrict__ out, int B, int H, int W,
                                    int P, int Hp, int Wp) {
  const int Kp = 3 * P * P;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * Hp * Wp * Kp) return;
  const long long patch = i / Kp;
  const int col = (int)(i % Kp), c = col / (P * P), py = (col / P) % P, px = col % P;
  const int pw = (int)(patch % Wp), ph = (int)((patch / Wp) % Hp), b = (int)(patch / ((long long)Wp * Hp));
  const int y = ph * P + py, x = pw * P + px;
  const float v = (y < H && x < W) ? pixel_value(img[(((long long)b * H + y) * W + x) * 3 + c], c) : 0.f;
  store_split(out + patch * 3 * Kp + col, Kp, 0, v);
}

// im2col of a ragged batch (vit.cu): imgs[b] gives image b's pixel offset, size, patch grid and first patch row.
// One thread = 8 consecutive pixels of one patch row, all three channels (the values and stores of im2col_f16_kernel,
// patch-major thread order); the split form writes one patch element per thread as im2col_split_kernel does. PAD: the
// ceil grid, a pixel outside the image is 0 (the values of im2col_f16_kernel<true> / im2col_split_kernel).
template <bool SPLIT, bool PAD>
__global__ void im2col_ragged_kernel(const uint8_t* __restrict__ img, __half* __restrict__ out,
                                     const RaggedImage* __restrict__ imgs, int B, long long n_patches, int P) {
  const int Kp = 3 * P * P, per_patch = SPLIT ? Kp : P * (P / 8);
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= n_patches * per_patch) return;
  const long long gp = gid / per_patch;                     // patch row of the packed batch
  const int r = (int)(gid % per_patch);
  const int b = ragged_find(B, gp, [&](int i) { return imgs[i].patch_off; });
  const RaggedImage im = imgs[b];
  const int n = (int)(gp - im.patch_off), ph = n / im.Wp, pw = n % im.Wp;
  if constexpr (SPLIT) {
    const int c = r / (P * P), y = ph * P + (r / P) % P, x = pw * P + r % P;
    const float v = (!PAD || (y < im.H && x < im.W)) ? pixel_value(img[(im.px_off + (long long)y * im.W + x) * 3 + c], c)
                                                      : 0.f;
    store_split(out + gp * 3 * Kp + r, Kp, 0, v);
  } else if constexpr (PAD) {
    const int py = r / (P / 8), px0 = (r % (P / 8)) * 8, y = ph * P + py, x0 = pw * P + px0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v[8];
#pragma unroll
      for (int t = 0; t < 8; ++t)
        v[t] = (y < im.H && x0 + t < im.W)
                   ? pixel_value(__ldg(img + (im.px_off + (long long)y * im.W + x0 + t) * 3 + c), c) : 0.f;
      uint4 q;
      q.x = pack_half2(v[0], v[1]);
      q.y = pack_half2(v[2], v[3]);
      q.z = pack_half2(v[4], v[5]);
      q.w = pack_half2(v[6], v[7]);
      *reinterpret_cast<uint4*>(out + gp * Kp + (c * P + py) * P + px0) = q;
    }
  } else {
    const int py = r / (P / 8), px0 = (r % (P / 8)) * 8;
    const uint8_t* src = img + (im.px_off + (long long)(ph * P + py) * im.W + pw * P + px0) * 3;
    uint8_t raw[24];
#pragma unroll
    for (int i = 0; i < 24; ++i) raw[i] = __ldg(src + i);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      uint4 q;
      q.x = pack_half2(pixel_value(raw[0 * 3 + c], c), pixel_value(raw[1 * 3 + c], c));
      q.y = pack_half2(pixel_value(raw[2 * 3 + c], c), pixel_value(raw[3 * 3 + c], c));
      q.z = pack_half2(pixel_value(raw[4 * 3 + c], c), pixel_value(raw[5 * 3 + c], c));
      q.w = pack_half2(pixel_value(raw[6 * 3 + c], c), pixel_value(raw[7 * 3 + c], c));
      *reinterpret_cast<uint4*>(out + gp * Kp + (c * P + py) * P + px0) = q;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, row kept in registers, two-pass variance (mean, then E[(x-mean)^2]) like torch,
// in the explicitly rounded arithmetic of the ln_* helpers (common.cuh). Output y [M, D] fp16, or with SPLIT the same
// fp32 value split in A order [M, 3D].
template <int D, bool SPLIT>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
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
  __half* yr = y + (long long)warp * (SPLIT ? 3 : 1) * D;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32 * i);
    const float4 bt = __ldg(reinterpret_cast<const float4*>(beta) + lane + 32 * i);
    const float4 o = ln_out4(v[i], rstd, g, bt);
    if constexpr (SPLIT) {
      __half* yc = yr + 4 * (lane + 32 * i);
      store_split(yc, D, 0, o.x);
      store_split(yc + 1, D, 0, o.y);
      store_split(yc + 2, D, 0, o.z);
      store_split(yc + 3, D, 0, o.w);
    } else {
      reinterpret_cast<uint2*>(yr)[lane + 32 * i] = make_uint2(pack_half2(o.x, o.y), pack_half2(o.z, o.w));
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// CLS row of the last block's attention (get_last_selfattention(...)[:, :, 0, 1:], the input of dino_seg):
// s_j = (q_0 . k_j) / 8 over all T tokens, softmax in fp32. One CTA per (head, image); the 64-term dot products are
// recomputed in each of the three passes (max, sum, output) rather than kept in scratch memory. KeyT: the qkv
// activations [M, 3d] of the fp16 path, or the fp32 qkv GEMM output of DSS_VIT_PRECISION_FP32. Loc (UniformRows /
// RaggedRows, common.cuh) says where image b's T_b tokens lie; its row of out is n_out long, the T_b - 1 patch entries
// and then exact zeros (n_out = T - 1 for a uniform batch).
constexpr int CLSATT_THREADS = 256;
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(float v) { return v; }
template <typename KeyT>
__device__ __forceinline__ float cls_score(const float* q0, const KeyT* k) {
  float acc = 0.f;
#pragma unroll 8
  for (int i = 0; i < 64; ++i) acc = fmaf(q0[i], to_f32(k[i]), acc);
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
template <typename KeyT, typename Loc>
__global__ void __launch_bounds__(CLSATT_THREADS)
cls_attention_kernel(const KeyT* __restrict__ qkv, Loc loc, int heads, int n_out, float* __restrict__ out) {
  __shared__ float q0[64];
  __shared__ float red[CLSATT_THREADS / 32 + 1];
  const int h = blockIdx.x, b = blockIdx.y, d = heads * 64, tid = threadIdx.x, T = loc.tokens(b);
  const KeyT* base = qkv + loc.row0(b) * 3 * d;
  const KeyT* kbase = base + d + h * 64;
  if (tid < 64) q0[tid] = to_f32(base[h * 64 + tid]);
  __syncthreads();
  float mx = -INFINITY;
  for (int j = tid; j < T; j += CLSATT_THREADS) mx = fmaxf(mx, cls_score(q0, kbase + (long long)j * 3 * d));
  mx = cls_block_reduce(mx, red, true);
  float sum = 0.f;
  for (int j = tid; j < T; j += CLSATT_THREADS) sum += expf(cls_score(q0, kbase + (long long)j * 3 * d) - mx);
  sum = cls_block_reduce(sum, red, false);
  float* o = out + ((long long)b * heads + h) * n_out;
  for (int j = tid + 1; j < T; j += CLSATT_THREADS) o[j - 1] = expf(cls_score(q0, kbase + (long long)j * 3 * d) - mx) / sum;
  for (int j = T - 1 + tid; j < n_out; j += CLSATT_THREADS) o[j] = 0.f;
}

// ---------------------------------------------------------------------------------------------------------------
// fp32 [rows, cols] -> split [rows, 3 cols], order 0 = A, 1 = B (the weights, once at load)
__global__ void split_rows_kernel(const float* __restrict__ x, __half* __restrict__ out, long long rows, int cols,
                                  int order) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const long long r = i / cols;
  const int c = (int)(i % cols);
  store_split(out + r * 3 * cols + c, cols, order, x[i]);
}

// MLP hidden activations: h [M, n] fp32 (fc1 output, bias included) -> gelu(h) in A order [M, 3n]. Exact erf, as
// torch's GELU: the polynomial gelu_erf of the fp16 path is accurate to 6.4e-6 only, an fp16-level error.
__global__ void gelu_split_kernel(const float* __restrict__ h, __half* __restrict__ out, long long M, int n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * n) return;
  const float x = h[i];
  const SplitF16 s = split_f16(0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)));
  store_split(out + (i / n) * 3 * n + (int)(i % n), n, 0, s.hi, s.hi_s, s.lo_s);
}

// qkv [M, 3d] fp32 (qkv GEMM output) -> per-head attention operands [M, 9d]: Q'_h at columns h*192 in A order, K'_h at
// 3d + h*192 and V'_h at 6d + h*192 in B order, 64 columns per group.
__global__ void qkv_split_kernel(const float* __restrict__ qkv, __half* __restrict__ out, long long M, int d) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * 3 * d) return;
  const long long r = i / (3 * d);
  const int c = (int)(i % (3 * d)), which = c / d, head = (c % d) >> 6, j = c & 63;
  store_split(out + r * 9 * d + (long long)which * 3 * d + head * 192 + j, 64, which, qkv[i]);
}

// ---------------------------------------------------------------------------------------------------------------
int launch_im2col(const uint8_t* img, void* patches, int B, int H, int W, int P, int pad, bool split, cudaStream_t st) {
  const char* name = split ? "im2col_split" : (pad ? "im2col_pad" : "im2col");
  DSS_REQUIRE(img && patches, "%s: null pointer", name);
  DSS_REQUIRE(P > 0 && (split || P % 8 == 0), "%s: patch must be a multiple of 8 (got %d)", name, P);
  DSS_REQUIRE(B > 0 && H > 0 && W > 0, "%s: empty image batch", name);
  const int Hp = pad ? cdiv(H, P) : H / P, Wp = pad ? cdiv(W, P) : W / P;
  DSS_REQUIRE(Hp > 0 && Wp > 0, "%s: image %dx%d smaller than one patch", name, H, W);
  __half* out = reinterpret_cast<__half*>(patches);
  LaunchScope scope(st, KC_IM2COL);
  if (split) {
    im2col_split_kernel<<<grid_for((long long)B * Hp * Wp * 3 * P * P, 256), 256, 0, st>>>(img, out, B, H, W, P, Hp, Wp);
  } else {
    const unsigned grid = grid_for((long long)B * Hp * Wp * P * (P / 8), 256);
    if (pad)
      im2col_f16_kernel<true><<<grid, 256, 0, st>>>(img, out, B, H, W, P, Hp, Wp);
    else
      im2col_f16_kernel<false><<<grid, 256, 0, st>>>(img, out, B, H, W, P, Hp, Wp);
  }
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_im2col_ragged(const uint8_t* img, void* patches, const RaggedImage* imgs, int B, long long n_patches, int P,
                         bool split, bool pad, cudaStream_t st) {
  DSS_REQUIRE(img && patches && imgs && B > 0 && n_patches > 0, "im2col_ragged: bad arguments");
  DSS_REQUIRE(P > 0 && P % 8 == 0, "im2col_ragged: patch must be a multiple of 8 (got %d)", P);
  __half* out = reinterpret_cast<__half*>(patches);
  const unsigned g_split = grid_for(n_patches * 3 * P * P, 256), g_f16 = grid_for(n_patches * P * (P / 8), 256);
  LaunchScope scope(st, KC_IM2COL);
  if (split && pad)
    im2col_ragged_kernel<true, true><<<g_split, 256, 0, st>>>(img, out, imgs, B, n_patches, P);
  else if (split)
    im2col_ragged_kernel<true, false><<<g_split, 256, 0, st>>>(img, out, imgs, B, n_patches, P);
  else if (pad)
    im2col_ragged_kernel<false, true><<<g_f16, 256, 0, st>>>(img, out, imgs, B, n_patches, P);
  else
    im2col_ragged_kernel<false, false><<<g_f16, 256, 0, st>>>(img, out, imgs, B, n_patches, P);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_layernorm(const float* x, const float* g, const float* b, void* y, int M, int d, float eps, bool split,
                     cudaStream_t st) {
  DSS_REQUIRE(d == 384 || d == 768, "layernorm: d must be 384 or 768 (got %d)", d);
  DSS_REQUIRE(M > 0, "layernorm: empty input");
  const int grid = cdiv(M, 8);  // 256 threads: 8 rows per CTA
  __half* yh = reinterpret_cast<__half*>(y);
  LaunchScope scope(st, KC_LAYERNORM);
  if (d == 384 && split)
    layernorm_kernel<384, true><<<grid, 256, 0, st>>>(x, g, b, yh, M, eps);
  else if (d == 384)
    layernorm_kernel<384, false><<<grid, 256, 0, st>>>(x, g, b, yh, M, eps);
  else if (split)
    layernorm_kernel<768, true><<<grid, 256, 0, st>>>(x, g, b, yh, M, eps);
  else
    layernorm_kernel<768, false><<<grid, 256, 0, st>>>(x, g, b, yh, M, eps);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_cls_attention(const void* qkv, bool f32_keys, int B, int T, int heads, float* out, cudaStream_t st) {
  DSS_REQUIRE(B > 0 && T >= 2 && heads > 0, "cls_attention: bad shape (B=%d T=%d heads=%d)", B, T, heads);
  const UniformRows loc{T, 0, 0, 0};
  LaunchScope scope(st, KC_ATTENTION);
  if (f32_keys)
    cls_attention_kernel<<<dim3(heads, B), CLSATT_THREADS, 0, st>>>(static_cast<const float*>(qkv), loc, heads, T - 1,
                                                                      out);
  else
    cls_attention_kernel<<<dim3(heads, B), CLSATT_THREADS, 0, st>>>(static_cast<const __half*>(qkv), loc, heads, T - 1,
                                                                      out);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_cls_attention_ragged(const void* qkv, bool f32_keys, const RaggedImage* imgs, int B, int n_out, int heads,
                                float* out, cudaStream_t st) {
  DSS_REQUIRE(qkv && imgs && out && B > 0 && n_out > 0 && heads > 0, "cls_attention_ragged: bad arguments");
  const RaggedRows loc{imgs, B};
  LaunchScope scope(st, KC_ATTENTION);
  if (f32_keys)
    cls_attention_kernel<<<dim3(heads, B), CLSATT_THREADS, 0, st>>>(static_cast<const float*>(qkv), loc, heads, n_out,
                                                                      out);
  else
    cls_attention_kernel<<<dim3(heads, B), CLSATT_THREADS, 0, st>>>(static_cast<const __half*>(qkv), loc, heads, n_out,
                                                                      out);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_split_rows(const float* x, void* out, long long rows, int cols, int order, cudaStream_t st, int kclass) {
  DSS_REQUIRE(x && out, "split: null pointer");
  DSS_REQUIRE(rows > 0 && cols > 0 && (order == 0 || order == 1), "split: bad arguments rows=%lld cols=%d order=%d",
              rows, cols, order);
  LaunchScope scope(st, kclass);
  split_rows_kernel<<<grid_for(rows * cols, 256), 256, 0, st>>>(x, reinterpret_cast<__half*>(out), rows, cols, order);
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

}  // namespace dss

using namespace dss;

extern "C" int dss_op_layernorm_f16(const float* x, const float* gamma, const float* beta, void* y, int M, int d,
                                    float eps, dss_stream_t stream) {
  return launch_layernorm(x, gamma, beta, y, M, d, eps, false, static_cast<cudaStream_t>(stream));
}
extern "C" int dss_op_layernorm_split_f16(const float* x, const float* gamma, const float* beta, void* y, int M, int d,
                                          float eps, dss_stream_t stream) {
  DSS_REQUIRE(x && gamma && beta && y, "layernorm_split: null pointer");
  return launch_layernorm(x, gamma, beta, y, M, d, eps, true, static_cast<cudaStream_t>(stream));
}
extern "C" int dss_op_im2col_f16(const uint8_t* images_u8, void* patches, int B, int H, int W, int P,
                                 dss_stream_t stream) {
  return launch_im2col(images_u8, patches, B, H, W, P, 0, false, static_cast<cudaStream_t>(stream));
}
extern "C" int dss_op_im2col_pad_f16(const uint8_t* images_u8, void* patches, int B, int H, int W, int P,
                                     dss_stream_t stream) {
  return launch_im2col(images_u8, patches, B, H, W, P, 1, false, static_cast<cudaStream_t>(stream));
}
extern "C" int dss_op_im2col_split_f16(const uint8_t* images_u8, void* patches, int B, int H, int W, int P, int pad,
                                       dss_stream_t stream) {
  return launch_im2col(images_u8, patches, B, H, W, P, pad, true, static_cast<cudaStream_t>(stream));
}
extern "C" int dss_op_cls_attention(const void* qkv, int B, int T, int heads, float* cls_attn, dss_stream_t stream) {
  DSS_REQUIRE(qkv && cls_attn, "cls_attention: null pointer");
  return launch_cls_attention(qkv, false, B, T, heads, cls_attn, static_cast<cudaStream_t>(stream));
}
extern "C" int dss_op_split_f16(const float* x, void* out, int rows, int cols, int order, dss_stream_t stream) {
  return launch_split_rows(x, out, rows, cols, order, static_cast<cudaStream_t>(stream), KC_MISC);
}
extern "C" int dss_op_gelu_split_f16(const float* h, void* out, int M, int n, dss_stream_t stream) {
  return launch_gelu_split(h, out, M, n, static_cast<cudaStream_t>(stream));
}
