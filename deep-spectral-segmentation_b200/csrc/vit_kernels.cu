// Non-GEMM kernels of the DINO ViT forward: pixel normalisation + im2col, CLS row, LayerNorm, attention.
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
// in the arithmetic of the ln_* helpers (common.cuh) that the fused LayerNorm GEMM shares.
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
// Attention, head dim 64: O = softmax(Q K^T / 8) V per (image, head), flash-style online softmax.
// CTA = 4 warps x 16 query rows; K/V streamed in 64-key tiles through a 2-stage cp.async ring;
// QK^T and PV on mma.sync m16n8k16 (fp16 in, fp32 accumulate); P never leaves registers.
// Shared tiles are [64 rows][64 halves] = 128 B rows with the 16 B chunk index XOR-swizzled by (row & 7).
constexpr int ATT_BM = 64, ATT_BN = 64, ATT_D = 64, ATT_THREADS = 128;

// loads a [64 x 64] half tile (rows row0.. of a [T, ld] matrix slice starting at column col0) with zero fill
__device__ __forceinline__ void att_load_tile(uint32_t tile_base, const __half* g, int row0, int T, long long ld,
                                              int tid) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = tid + i * ATT_THREADS;  // 0..511
    const int r = idx >> 3, ch = idx & 7;
    const bool ok = (row0 + r) < T;
    const __half* src = g + (long long)(ok ? row0 + r : 0) * ld + ch * 8;
    cp_async_16(sw128_addr(tile_base, r, ch), src, ok);
  }
}

__global__ void __launch_bounds__(ATT_THREADS)
attention_f16_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int T, int heads) {
  __shared__ __align__(128) uint8_t smem[(1 + 2 + 2) * ATT_BM * ATT_D * 2];  // Q | K0 K1 | V0 V1 = 40 KB
  const int d = heads * ATT_D;
  const long long ld = 3LL * d;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const __half* qg = qkv + (long long)b * T * ld + h * ATT_D;
  const __half* kg = qg + d;
  const __half* vg = qg + 2 * d;
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK = sQ + ATT_BM * ATT_D * 2;
  const uint32_t sV = sK + 2 * ATT_BN * ATT_D * 2;
  const int q0 = qt * ATT_BM;
  const int ntiles = (T + ATT_BN - 1) / ATT_BN;

  att_load_tile(sQ, qg, q0, T, ld, tid);
  att_load_tile(sK, kg, 0, T, ld, tid);
  att_load_tile(sV, vg, 0, T, ld, tid);
  cp_async_commit();

  // softmax in base 2: p = 2^(s*c - m*c), c = log2(e)/sqrt(64)
  const float sc = 1.4426950408889634f * 0.125f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};
  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  uint32_t qf[4][4];

  for (int j = 0; j < ntiles; ++j) {
    const int st = j & 1;
    if (j + 1 < ntiles) {
      att_load_tile(sK + (st ^ 1) * ATT_BN * ATT_D * 2, kg, (j + 1) * ATT_BN, T, ld, tid);
      att_load_tile(sV + (st ^ 1) * ATT_BN * ATT_D * 2, vg, (j + 1) * ATT_BN, T, ld, tid);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (j == 0) {
      // Q fragments (A operand, 16 rows of this warp x 64) stay in registers for the whole kernel
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const int r = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        const int ch = ks * 2 + (lane >> 4);
        ldmatrix_x4(sw128_addr(sQ, r, ch), qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
      }
    }
    const uint32_t kt = sK + st * ATT_BN * ATT_D * 2;
    const uint32_t vt = sV + st * ATT_BN * ATT_D * 2;

    // S = Q K^T : 8 n-tiles (8 keys each) x 4 k-steps
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {  // pairs of n-tiles
        uint32_t b0, b1, b2, b3;
        const int r = np * 16 + (lane & 7) + (lane >> 4) * 8;  // key row
        const int ch = ks * 2 + ((lane >> 3) & 1);
        ldmatrix_x4(sw128_addr(kt, r, ch), b0, b1, b2, b3);
        mma_m16n8k16_f16(s[np * 2], qf[ks], b0, b1);
        mma_m16n8k16_f16(s[np * 2 + 1], qf[ks], b2, b3);
      }
    }
    // mask keys beyond T (only the last tile can be partial)
    const int kbase = j * ATT_BN;
    if (kbase + ATT_BN > T) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int key = kbase + i * 8 + (lane & 3) * 2;
        if (key >= T) s[i][0] = s[i][2] = -INFINITY;
        if (key + 1 >= T) s[i][1] = s[i][3] = -INFINITY;
      }
    }
    // online softmax; thread owns rows (lane/4) [regs 0,1] and (lane/4 + 8) [regs 2,3]
    float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      mx[0] = fmaxf(mx[0], fmaxf(s[i][0], s[i][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[i][2], s[i][3]));
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
    float corr[2], msc[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      corr[r] = exp2f((m_run[r] - mx[r]) * sc);  // first tile: exp2(-inf) = 0
      m_run[r] = mx[r];
      msc[r] = mx[r] * sc;
      l_run[r] *= corr[r];
    }
    float rs[2] = {0.f, 0.f};
    uint32_t pf[4][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float p0 = exp2f(fmaf(s[i][0], sc, -msc[0]));
      const float p1 = exp2f(fmaf(s[i][1], sc, -msc[0]));
      const float p2 = exp2f(fmaf(s[i][2], sc, -msc[1]));
      const float p3 = exp2f(fmaf(s[i][3], sc, -msc[1]));
      rs[0] += p0 + p1;
      rs[1] += p2 + p3;
      // accumulator layout of two adjacent n-tiles == A-operand layout of one 16-wide k-step
      pf[i >> 1][(i & 1) * 2 + 0] = pack_half2(p0, p1);
      pf[i >> 1][(i & 1) * 2 + 1] = pack_half2(p2, p3);
    }
    l_run[0] += rs[0];
    l_run[1] += rs[1];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[i][0] *= corr[0]; o[i][1] *= corr[0];
      o[i][2] *= corr[1]; o[i][3] *= corr[1];
    }
    // O += P V : 4 k-steps (16 keys) x 8 n-tiles (8 head dims); V read transposed by ldmatrix
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t b0, b1, b2, b3;
        const int r = ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;  // key row
        const int ch = np * 2 + (lane >> 4);                          // head-dim chunk
        ldmatrix_x4_trans(sw128_addr(vt, r, ch), b0, b1, b2, b3);
        mma_m16n8k16_f16(o[np * 2], pf[ks], b0, b1);
        mma_m16n8k16_f16(o[np * 2 + 1], pf[ks], b2, b3);
      }
    }
    __syncthreads();  // all warps done with stage `st` before it is refilled
  }

  // finalise: row sums across the 4 lanes of a quad, normalise, store f16
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const float inv0 = 1.0f / l_run[0], inv1 = 1.0f / l_run[1];
  const int row0 = q0 + warp * 16 + (lane >> 2);
  __half* og = out + (long long)b * T * d + h * ATT_D + (lane & 3) * 2;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (row0 < T)
      *reinterpret_cast<uint32_t*>(og + (long long)row0 * d + i * 8) = pack_half2(o[i][0] * inv0, o[i][1] * inv0);
    if (row0 + 8 < T)
      *reinterpret_cast<uint32_t*>(og + (long long)(row0 + 8) * d + i * 8) = pack_half2(o[i][2] * inv1, o[i][3] * inv1);
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

int launch_attention(const void* qkv, void* out, int B, int T, int heads, cudaStream_t st) {
  DSS_REQUIRE(B > 0 && T > 0 && heads > 0, "attention: empty problem");
  dim3 grid(cdiv(T, ATT_BM), heads, B);
  LaunchScope scope(st, KC_ATTENTION);
  attention_f16_kernel<<<grid, ATT_THREADS, 0, st>>>(reinterpret_cast<const __half*>(qkv),
                                                     reinterpret_cast<__half*>(out), T, heads);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

}  // namespace dss

using namespace dss;

extern "C" int dss_op_layernorm_f16(const float* x, const float* gamma, const float* beta, void* y, int M, int d,
                                    float eps, dss_stream_t stream) {
  return launch_layernorm(x, gamma, beta, y, M, d, eps, static_cast<cudaStream_t>(stream));
}
extern "C" int dss_op_attention_f16(const void* qkv, void* out, int B, int T, int heads, dss_stream_t stream) {
  return launch_attention(qkv, out, B, T, heads, static_cast<cudaStream_t>(stream));
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
