// DINO ViT feature extractor: weight packing, positional-embedding interpolation, forward orchestration.
// Replaces utils.get_model + model.get_intermediate_layers + the qkv forward hook of the reference
// (extract/extract_utils.py:40-50, extract/extract.py:49-53,82-98).
//
// Per block:  LN1 -> [wgmma GEMM] qkv (f16) -> wgmma flash attention -> [wgmma GEMM + residual] proj
//             LN2 -> [wgmma GEMM + GELU] fc1 (f16) -> [wgmma GEMM + residual] fc2
// The residual stream stays fp32; GEMM operands are fp16 (11-bit significand, same as TF32), accumulation fp32.
// DSS_VIT_PRECISION_FP32 (dss_vit_set_precision) runs the same blocks on split-fp16 operands (the split producers of
// vit_kernels.cu, attention_split_kernel): fp32-equivalent products on the fp16 tensor cores at three times the
// tensor-core work.
// The block the reference hooks is pruned to LN1 + the K third of its qkv projection, CLS row dropped in the
// GEMM epilogue, which writes the fp32 features directly in the reference's [B, N, d] layout.
#include <limits.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <cstring>
#include <utility>
#include <vector>

#include "common.cuh"

namespace dss {

// y[b, :] = LayerNorm(x[row0(b), :]) * gamma + beta in fp32 (one warp per image): the final norm of the CLS token, read
// where it lies in the residual stream
template <typename Loc>
__global__ void __launch_bounds__(128)
layernorm_rows_f32_kernel(const float* __restrict__ x, Loc loc, const float* __restrict__ gamma,
                          const float* __restrict__ beta, float* __restrict__ y, int rows, int d, float eps) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + loc.row0(row) * d;
  float s = 0.f;
  for (int i = lane; i < d; i += 32) s += xr[i];
  const float mean = warp_sum(s) / (float)d;
  float q = 0.f;
  for (int i = lane; i < d; i += 32) { const float a = xr[i] - mean; q = fmaf(a, a, q); }
  const float rstd = rsqrtf(warp_sum(q) / (float)d + eps);
  for (int i = lane; i < d; i += 32) y[(long long)row * d + i] = (xr[i] - mean) * rstd * gamma[i] + beta[i];
}

__global__ void f32_to_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = __float2half_rn(src[i]);
}

struct BlockW {
  float *ln1_w, *ln1_b, *ln2_w, *ln2_b, *qkv_b, *proj_b, *fc1_b, *fc2_b;
  __half *qkv_w, *proj_w, *fc1_w, *fc2_w;
  CUtensorMap tm_qkv, tm_k, tm_proj, tm_fc1, tm_fc2;
  CUtensorMap tm_q, tm_v;             // q and v thirds of the qkv weight (localization features)
};

}  // namespace dss

struct dss_vit {
  dss_vit_config cfg;
  int precision = DSS_VIT_PRECISION_FP16;   // DSS_VIT_PRECISION_FP32: every weight packed as split fp16 (B order)
  bool loaded = false;
  void* arena = nullptr;  // one device allocation holding every packed weight
  size_t arena_bytes = 0;
  __half* patch_w = nullptr;
  float *patch_b = nullptr, *cls = nullptr;
  float *norm_w = nullptr, *norm_b = nullptr;   // final LayerNorm (only needed by dss_vit_forward_cls)
  float* pos_dev = nullptr;   // [1 + grid0^2, d] the stored positional grid (every forward interpolates it on the device)
  CUtensorMap tm_patch;
  std::vector<dss::BlockW> blocks;
};

namespace dss {

// ---- bicubic interpolation of the positional grid exactly as torch F.interpolate(mode='bicubic',
// align_corners=False, scale_factor=s) computes it: src = (dst + 0.5) / s - 0.5, A = -0.75, border clamp.
static inline double cubic1(double x, double A) { return ((A + 2.0) * x - (A + 3.0)) * x * x + 1.0; }
static inline double cubic2(double x, double A) { return ((A * x - 5.0 * A) * x + 8.0 * A) * x - 4.0 * A; }

static void interp_axis(int in, int out, double scale_factor, std::vector<int>& idx, std::vector<float>& w) {
  idx.resize(out);
  w.resize((size_t)out * 4);
  const double A = -0.75;
  const float rscale = (float)(1.0 / scale_factor);  // torch keeps the scale in fp32 for fp32 inputs
  for (int o = 0; o < out; ++o) {
    const float real = rscale * ((float)o + 0.5f) - 0.5f;
    const float fl = floorf(real);
    const double t = (double)(real - fl);
    idx[o] = (int)fl;
    w[o * 4 + 0] = (float)cubic2(t + 1.0, A);
    w[o * 4 + 1] = (float)cubic1(t, A);
    w[o * 4 + 2] = (float)cubic1(1.0 - t, A);
    w[o * 4 + 3] = (float)cubic2(2.0 - t, A);
  }
  (void)in;
}

// Upstream interpolate_pos_encoding returns the stored grid only when npatch == N0 and the input's PIXEL height equals
// its width. A g x g patch grid from a non-square input (a 224 x 232 box crop at patch 16) is still resampled, with
// scale (g + 0.1) / g, which is not the identity. `square`: the input's pixel sizes are equal, or the caller crops to
// patch multiples first as the reference does before get_intermediate_layers (then Hp == Wp decides).
static bool pos_is_stored(int g, int Hp, int Wp, bool square) { return Hp == g && Wp == g && square; }

// The identity rule for one H x W image with an Hp x Wp patch grid. The model's own forward (the final-norm CLS token
// and the residual-stream hook) takes the image as is, so its pixel sizes decide; forward_k's and localization's inputs
// are cropped or padded to patch multiples by the reference before the model sees them, so their patch grid decides.
static bool image_pos_is_stored(int g, int H, int W, int Hp, int Wp, bool own_forward) {
  return pos_is_stored(g, Hp, Wp, own_forward ? H == W : Hp == Wp);
}

// pos_src [1 + g*g, d] -> pos_out [1 + Hp*Wp, d]; host memory, pure CPU: the reference the device tables (pos_cls_kernel)
// are tested against
static void interp_pos_host(const float* src, int g, int d, int Hp, int Wp, bool square, float* pos) {
  std::copy(src, src + d, pos);  // CLS slot untouched
  if (pos_is_stored(g, Hp, Wp, square)) {
    std::copy(src + d, src + (size_t)(g * g + 1) * d, pos + d);
    return;
  }
  // upstream: scale_factor = ((Hp + 0.1) / sqrt(N0), (Wp + 0.1) / sqrt(N0)); output size floor(g * scale) == Hp, Wp
  std::vector<int> iy, ix;
  std::vector<float> wy, wx;
  interp_axis(g, Hp, ((double)Hp + 0.1) / (double)g, iy, wy);
  interp_axis(g, Wp, ((double)Wp + 0.1) / (double)g, ix, wx);
  auto clampi = [g](int v) { return v < 0 ? 0 : (v >= g ? g - 1 : v); };
  for (int y = 0; y < Hp; ++y)
    for (int x = 0; x < Wp; ++x) {
      float* o = pos + ((size_t)(y * Wp + x) + 1) * d;
      for (int c = 0; c < d; ++c) o[c] = 0.f;
      for (int a = 0; a < 4; ++a) {
        const int sy = clampi(iy[y] - 1 + a);
        for (int b = 0; b < 4; ++b) {
          const int sx = clampi(ix[x] - 1 + b);
          const float wgt = wy[y * 4 + a] * wx[x * 4 + b];
          const float* s = src + ((size_t)(sy * g + sx) + 1) * d;
          for (int c = 0; c < d; ++c) o[c] += wgt * s[c];
        }
      }
    }
}

// ---- the same interpolation on the device. interp_axis's taps for output cell o of an axis of n cells: the scale, its
// reciprocal and the cubic coefficients in double and the source coordinate in fp32, every operation rounded on its
// own as the host code rounds it (no contraction), so the taps are the host's bits. Returns the first source index.
__device__ __forceinline__ double cubic1_rn(double x, double A) {
  return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(A + 2.0, x), A + 3.0), x), x), 1.0);
}
__device__ __forceinline__ double cubic2_rn(double x, double A) {
  return __dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(__dmul_rn(A, x), 5.0 * A), x), 8.0 * A), x), 4.0 * A);
}
__device__ __forceinline__ int pos_taps(int g, int n, int o, float (&w)[4]) {
  const double A = -0.75;
  const float rscale = __double2float_rn(__ddiv_rn(1.0, __ddiv_rn(__dadd_rn((double)n, 0.1), (double)g)));
  const float real = __fsub_rn(__fmul_rn(rscale, __fadd_rn((float)o, 0.5f)), 0.5f);
  const float fl = floorf(real);
  const double t = (double)__fsub_rn(real, fl);
  w[0] = __double2float_rn(cubic2_rn(__dadd_rn(t, 1.0), A));
  w[1] = __double2float_rn(cubic1_rn(t, A));
  w[2] = __double2float_rn(cubic1_rn(__dsub_rn(1.0, t), A));
  w[3] = __double2float_rn(cubic2_rn(__dsub_rn(2.0, t), A));
  return (int)fl;
}

// The token embedding's shape-dependent part, before the patch GEMM: the positional table pos [rows, d] (Loc: one
// shared [T, d] table, or a ragged batch's tables laid out like the residual stream) and every image's CLS row
// x[row0(b)] = cls + pos[0]. The bicubic resampling of interp_pos_host with the same tap order and every product and
// sum rounded on its own, so the tables are dss_pos_embed_interp_host's bits; the CLS slot and, under the identity
// rule, the whole grid are copied. One thread per POS_PC consecutive channels of max(rows, B) rows (d is 384 or 768),
// so the taps are computed once for POS_PC outputs.
constexpr int POS_PC = 4;
template <typename Loc>
__global__ void pos_cls_kernel(const float* __restrict__ grid, int g, const float* __restrict__ cls, Loc loc, int B,
                               long long rows, int d, float* __restrict__ pos, float* __restrict__ x) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * POS_PC;
  const long long r = i / d;
  const int c0 = (int)(i % d);
  if (r < B) {
#pragma unroll
    for (int c = c0; c < c0 + POS_PC; ++c) x[loc.row0((int)r) * d + c] = cls[c] + grid[c];
  }
  if (r >= rows) return;
  const PosRow p = loc.at(r);
  if (p.t == 0 || p.stored) {
#pragma unroll
    for (int k = 0; k < POS_PC; ++k) pos[i + k] = grid[(long long)p.t * d + c0 + k];
    return;
  }
  float wy[4], wx[4];
  const int iy = pos_taps(g, p.Hp, (p.t - 1) / p.Wp, wy), ix = pos_taps(g, p.Wp, (p.t - 1) % p.Wp, wx);
  float o[POS_PC] = {};
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int sy = min(max(iy - 1 + a, 0), g - 1);
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int sx = min(max(ix - 1 + b, 0), g - 1);
      const float wgt = __fmul_rn(wy[a], wx[b]);
      const float* s = grid + ((long long)(sy * g + sx) + 1) * d + c0;
#pragma unroll
      for (int k = 0; k < POS_PC; ++k) o[k] = __fadd_rn(o[k], __fmul_rn(wgt, s[k]));
    }
  }
#pragma unroll
  for (int k = 0; k < POS_PC; ++k) pos[i + k] = o[k];
}

// ks = 1 (DSS_VIT_PRECISION_FP16) or 3 (DSS_VIT_PRECISION_FP32, split): patches, xn and attn hold ks fp16 groups per
// value (A order). Split, qkv holds the split attention operands [B*T, 9d] and, after attention, the split MLP hidden
// activations [B*T, 12d] (the same buffer), and f32 holds the fp32 GEMM outputs that are split next: qkv [B*T, 3d],
// then the fc1 output [B*T, 4d].
struct VitWs {
  __half* patches;  // [B*Np, ks 3P^2]
  float* x;         // [B*T, d]     residual stream
  __half* xn;       // [B*T, ks d]  LayerNorm output (GEMM A operand)
  __half* attn;     // [B*T, ks d]  attention output (GEMM A operand)
  __half* qkv;      // [B*T, 3d] (fp16) | [B*T, 9d] (split)
  __half* hid;      // [B*T, ks 4d]
  float* f32;       // split only
  float* pos;       // [pos_rows, d] positional table(s)
  size_t total;
};

// n_patches patch rows and M token rows (B Np and B T for a uniform batch); pos_rows positional rows (T for a uniform
// batch, whose images share one table; M for a ragged one)
static VitWs carve(const dss_vit_config& c, size_t n_patches, size_t M, size_t pos_rows, void* base, int precision) {
  const int d = c.dim;
  const size_t ks = precision == DSS_VIT_PRECISION_FP32 ? 3 : 1;
  uint8_t* p = reinterpret_cast<uint8_t*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint8_t* r = p ? p + off : nullptr;
    off += align_up(bytes, 1024);
    return r;
  };
  VitWs w;
  const size_t hd = (size_t)c.mlp_ratio * d;
  w.patches = reinterpret_cast<__half*>(take(n_patches * ks * 3 * c.patch * c.patch * 2));
  w.x = reinterpret_cast<float*>(take(M * d * 4));
  w.xn = reinterpret_cast<__half*>(take(M * ks * d * 2));
  w.attn = reinterpret_cast<__half*>(take(M * ks * d * 2));
  const size_t qkv_bytes = M * ks * 3 * d * 2, hid_bytes = M * ks * hd * 2;
  if (ks == 3) {
    w.qkv = w.hid = reinterpret_cast<__half*>(take(std::max(qkv_bytes, hid_bytes)));
    w.f32 = reinterpret_cast<float*>(take(M * std::max<size_t>(3 * d, hd) * 4));
  } else {
    w.qkv = reinterpret_cast<__half*>(take(qkv_bytes));
    w.hid = reinterpret_cast<__half*>(take(hid_bytes));
    w.f32 = nullptr;
  }
  w.pos = reinterpret_cast<float*>(take(pos_rows * d * 4));
  w.total = off;
  return w;
}

// A ragged batch as vit_run sees it: B images of any sizes, n_patches patch rows and M token rows packed image after
// image, and the device tables (in the workspace) that the shape-dependent kernels read.
struct Ragged {
  int B;
  long long n_patches, M;
  int tiles;                      // 128-query attention tiles over all images
  const RaggedImage* imgs;        // [B]
  const int* tile_prefix;         // [B + 1]
  const int* patch_rows;          // [n_patches] token row of each patch row
  const int* k_rows;              // [M] feature row of each token row (-1: CLS)
  int n_out;                      // feature rows per image of a padded output [B, n_out, d] (0: packed output)
};

// the positional table (pos_rows rows) and every image's CLS row: pos_cls_kernel over batch `loc`
template <typename Loc>
static int launch_pos_cls(const dss_vit* h, Loc loc, int B, long long pos_rows, const VitWs& w, cudaStream_t st) {
  const int d = h->cfg.dim;
  const long long n = std::max<long long>(pos_rows, B) * (d / POS_PC);
  LaunchScope scope(st, KC_CLS_ROW);
  pos_cls_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(h->pos_dev, h->cfg.grid0, h->cls, loc, B, pos_rows, d,
                                                              w.pos, w.x);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

// modes 1 and 2 after the blocks: the residual stream, or the final LayerNorm of the CLS rows
static int vit_tail(const dss_vit* h, const float* x, int mode, float* out, int B, const UniformRows& uni,
                    const Ragged* rg, cudaStream_t st) {
  const int d = h->cfg.dim;
  if (mode == 2) {
    // upstream VisionTransformer.forward: x = norm(x); return x[:, 0]  (LayerNorm is row-wise: only the CLS rows)
    DSS_REQUIRE(h->norm_w && h->norm_b, "vit: the final LayerNorm weights (norm.weight / norm.bias) were not loaded");
    LaunchScope scope(st, KC_LAYERNORM);
    if (rg)
      layernorm_rows_f32_kernel<<<cdiv(B, 4), 128, 0, st>>>(x, RaggedRows{rg->imgs, B}, h->norm_w, h->norm_b, out, B, d,
                                                            h->cfg.ln_eps);
    else
      layernorm_rows_f32_kernel<<<cdiv(B, 4), 128, 0, st>>>(x, uni, h->norm_w, h->norm_b, out, B, d, h->cfg.ln_eps);
    DSS_CHECK_CUDA(cudaGetLastError());
  } else {
    DSS_REQUIRE(!rg, "vit: no residual-stream output for ragged batches");
    DSS_CHECK_CUDA(cudaMemcpyAsync(out, x, (size_t)B * uni.T * d * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  return DSS_OK;
}

// mode 0: K projection of block n_full (features), 1: residual stream [B, T, d], 2: final-norm CLS token [B, d],
// 3: block n_full's `which` projection third (out, may be NULL) and CLS attention row (cls_attn, may be NULL); mode 0
// is mode 3 with which = 1 and no CLS attention row. pad: zero-padded ceil grid instead of the crop.
// DSS_VIT_PRECISION_FP32 runs the same sequence on split operands: every GEMM runs the fp16 path's kernel and epilogue
// at K' = 3 K; the qkv and fc1 GEMMs write fp32 (DSS_EPI_BIAS_F32), which qkv_split_kernel / gelu_split_kernel turn
// into the next product's split operands.
// rg: a ragged batch (modes 0, 2 and 3; H, W unused). Only the token embedding, attention, the projection's CLS drop,
// the CLS attention row and the final-norm rows depend on image boundaries; they read rg's tables, every other step is
// row-wise over M rows. Mode 3 writes rg's padded layout: out [B, n_out, d] and cls_attn [B, heads, n_out], the rows
// past an image's N_b exact zeros.
static int vit_run(dss_vit* h, const uint8_t* img, int B, int H, int W, int n_full, int mode, float* out, void* ws,
                   size_t ws_bytes, cudaStream_t st, int pad = 0, int which = 1, float* cls_attn = nullptr,
                   const Ragged* rg = nullptr) {
  DSS_REQUIRE(h && h->loaded, "vit: weights not loaded");
  DSS_REQUIRE(img && (out || cls_attn) && ws, "vit: null pointer");
  const dss_vit_config& c = h->cfg;
  const int P = c.patch, d = c.dim, hd = c.mlp_ratio * d;
  const int Hp = rg ? 0 : (pad ? cdiv(H, P) : H / P), Wp = rg ? 0 : (pad ? cdiv(W, P) : W / P);
  DSS_REQUIRE(rg || (B > 0 && Hp > 0 && Wp > 0), "vit: image %dx%d smaller than one %d-pixel patch", H, W, P);
  DSS_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "vit: workspace must be 256-byte aligned");
  const int Np = Hp * Wp, T = Np + 1, Kp = 3 * P * P;
  const int M = rg ? (int)rg->M : B * T, n_patches = rg ? (int)rg->n_patches : B * Np;
  const bool split = h->precision == DSS_VIT_PRECISION_FP32;
  const int ks = split ? 3 : 1;   // fp16 values per operand value
  VitWs w = carve(c, (size_t)n_patches, (size_t)M, rg ? (size_t)M : (size_t)T, ws, h->precision);
  if (ws_bytes < w.total) {
    set_error("vit: workspace too small (%zu < %zu)", ws_bytes, w.total);
    return DSS_ERR_WORKSPACE;
  }
  const UniformRows uni{T, Hp, Wp, !rg && image_pos_is_stored(c.grid0, H, W, Hp, Wp, mode == 1 || mode == 2)};
  int rc;

  CUtensorMap tm_patches, tm_xn, tm_attn, tm_hid;
  if ((rc = make_tmap_f16(&tm_patches, w.patches, n_patches, ks * Kp, 128))) return rc;
  if ((rc = make_tmap_f16(&tm_xn, w.xn, M, ks * d, 128))) return rc;
  if ((rc = make_tmap_f16(&tm_attn, w.attn, M, ks * d, 128))) return rc;
  if ((rc = make_tmap_f16(&tm_hid, w.hid, M, ks * hd, 128))) return rc;
  // output maps of the TMA-store epilogues: residual stream (fp32, reduce-add), qkv and MLP hidden (fp16, or the fp32
  // outputs that are split next)
  CUtensorMap tm_x_out, tm_qkv_out, tm_hid_out;
  if ((rc = make_tmap_out(&tm_x_out, w.x, M, d, 1))) return rc;
  if ((rc = make_tmap_out(&tm_qkv_out, split ? (void*)w.f32 : w.qkv, M, 3 * d, split))) return rc;
  if ((rc = make_tmap_out(&tm_hid_out, split ? (void*)w.f32 : w.hid, M, hd, split))) return rc;

  // tokens: x[b, 0, :] = cls + pos[0] and the positional table, then x[b, 1+n, :] = patch_embed + pos[1+n]
  if (rg) {
    if ((rc = launch_im2col_ragged(img, w.patches, rg->imgs, B, n_patches, P, split, pad, st))) return rc;
    if ((rc = launch_pos_cls(h, RaggedRows{rg->imgs, B}, B, M, w, st))) return rc;
    if ((rc = gemm_f16_tc_rows(tm_patches, h->tm_patch, h->patch_b, w.x, n_patches, d, ks * Kp, DSS_EPI_PATCH_F32,
                               w.pos, rg->patch_rows, st, KC_GEMM_PATCH)))
      return rc;
  } else {
    if ((rc = launch_im2col(img, w.patches, B, H, W, P, pad, split, st))) return rc;
    if ((rc = launch_pos_cls(h, uni, B, T, w, st))) return rc;
    if ((rc = gemm_f16_tc(tm_patches, h->tm_patch, nullptr, h->patch_b, w.x, n_patches, d, ks * Kp, DSS_EPI_PATCH_F32,
                          w.pos, Np, T, st, KC_GEMM_PATCH, 128)))
      return rc;
  }

  // the full qkv projection: the attention operands (fp16), or the fp32 values they are split from
  auto qkv_gemm = [&](const BlockW& bw) {
    return gemm_f16_tc(tm_xn, bw.tm_qkv, &tm_qkv_out, bw.qkv_b, split ? (void*)w.f32 : w.qkv, M, 3 * d, ks * d,
                       split ? DSS_EPI_BIAS_F32 : DSS_EPI_BIAS_F16, nullptr, 0, 0, st, KC_GEMM_QKV, gemm_tile_n());
  };
  auto attention = [&]() {
    if (split) {
      if ((rc = launch_qkv_split(w.f32, w.qkv, M, d, st))) return rc;
      return rg ? launch_attention_split_ragged(w.qkv, w.attn, rg->imgs, rg->tile_prefix, B, M, rg->tiles, c.heads, st)
                : launch_attention_split(w.qkv, w.attn, B, T, c.heads, st);
    }
    return rg ? launch_attention_tc_ragged(w.qkv, w.attn, rg->imgs, rg->tile_prefix, B, M, rg->tiles, c.heads, st)
              : launch_attention_tc(w.qkv, w.attn, B, T, c.heads, st);
  };
  // LayerNorm kernel + GEMM: LayerNorm fused into the qkv / fc1 GEMMs measured slower (DESIGN.md section 9)
  for (int l = 0; l < n_full; ++l) {
    const BlockW& bw = h->blocks[l];
    if ((rc = launch_layernorm(w.x, bw.ln1_w, bw.ln1_b, w.xn, M, d, c.ln_eps, split, st))) return rc;
    if ((rc = qkv_gemm(bw))) return rc;
    if ((rc = attention())) return rc;
    if ((rc = gemm_f16_tc(tm_attn, bw.tm_proj, &tm_x_out, bw.proj_b, w.x, M, d, ks * d, DSS_EPI_BIAS_RESID_F32, nullptr,
                          0, 0, st, KC_GEMM_PROJ, gemm_tile_n())))
      return rc;
    if ((rc = launch_layernorm(w.x, bw.ln2_w, bw.ln2_b, w.xn, M, d, c.ln_eps, split, st))) return rc;
    if ((rc = gemm_f16_tc(tm_xn, bw.tm_fc1, &tm_hid_out, bw.fc1_b, split ? (void*)w.f32 : w.hid, M, hd, ks * d,
                          split ? DSS_EPI_BIAS_F32 : DSS_EPI_BIAS_GELU_F16, nullptr, 0, 0, st, KC_GEMM_FC1,
                          gemm_tile_n())))
      return rc;
    if (split && (rc = launch_gelu_split(w.f32, w.hid, M, hd, st))) return rc;
    if ((rc = gemm_f16_tc(tm_hid, bw.tm_fc2, &tm_x_out, bw.fc2_b, w.x, M, d, ks * hd, DSS_EPI_BIAS_RESID_F32, nullptr, 0,
                          0, st, KC_GEMM_FC2, gemm_tile_n())))
      return rc;
  }
  if (mode == 1 || mode == 2) return vit_tail(h, w.x, mode, out, B, uni, rg, st);

  const BlockW& bw = h->blocks[n_full];
  if ((rc = launch_layernorm(w.x, bw.ln1_w, bw.ln1_b, w.xn, M, d, c.ln_eps, split, st))) return rc;
  if (out) {   // qkv[b, 1+n, which*d : (which+1)*d] in fp32, CLS rows dropped (which = 1: the K features)
    const CUtensorMap& tm = which == 0 ? bw.tm_q : (which == 1 ? bw.tm_k : bw.tm_v);
    // the rows of a padded output that no token row maps to
    if (rg && rg->n_out) DSS_CHECK_CUDA(cudaMemsetAsync(out, 0, (size_t)B * rg->n_out * d * sizeof(float), st));
    rc = rg ? gemm_f16_tc_rows(tm_xn, tm, bw.qkv_b + (size_t)which * d, out, M, d, ks * d, DSS_EPI_DROPCLS_F32, nullptr,
                               rg->k_rows, st, KC_GEMM_KPROJ)
            : gemm_f16_tc(tm_xn, tm, nullptr, bw.qkv_b + (size_t)which * d, out, M, d, ks * d, DSS_EPI_DROPCLS_F32,
                          nullptr, T, Np, st, KC_GEMM_KPROJ, 128);
    if (rc) return rc;
  }
  if (cls_attn) {   // the full qkv projection the attention kernels read, then the CLS row of the softmax
    if ((rc = qkv_gemm(bw))) return rc;
    const void* keys = split ? (const void*)w.f32 : w.qkv;
    rc = rg ? launch_cls_attention_ragged(keys, split, rg->imgs, B, rg->n_out, c.heads, cls_attn, st)
            : launch_cls_attention(keys, split, B, T, c.heads, cls_attn, st);
    if (rc) return rc;
  }
  return DSS_OK;
}

// ---- ragged batches: host plan. Workspace = the forward's buffers (carve, positional tables [M, d] included) | one
// block of tables (RaggedImage [B], tile_prefix [B + 1], patch_rows [n_patches], k_rows [M]), uploaded with one copy
// per forward. Mode DSS_VIT_RAGGED_PAD runs the zero-padded ceil grid of forward_last(pad = 1), so an image may be
// smaller than one patch; the others crop.
struct RaggedPlan {
  std::vector<RaggedImage> imgs;
  std::vector<int> tile_prefix, patch_rows, k_rows;
  long long n_patches = 0, M = 0;
  size_t vit_bytes = 0, tables_bytes = 0, total = 0;
  size_t t_imgs = 0, t_tiles = 0, t_prows = 0, t_krows = 0;   // offsets inside the table block
};

constexpr int RAGGED_TILE = 128;   // query rows per attention CTA (FA_BM, AS_BM)

// Validates the batch and lays out its workspace; with `tables`, also fills the host tables. mode: DSS_VIT_RAGGED_*.
// n_out > 0: the features go to a padded [B, n_out, d] output (image b's row n at b n_out + n), which must hold every
// image's N_b rows; 0: packed.
static int ragged_plan(const dss_vit* h, const int* dims, int B, int mode, int n_out, bool tables, RaggedPlan& pl) {
  DSS_REQUIRE(h && dims, "vit_ragged: null pointer");
  DSS_REQUIRE(B > 0, "vit_ragged: B must be positive (got %d)", B);
  DSS_REQUIRE(mode == DSS_VIT_RAGGED_K || mode == DSS_VIT_RAGGED_CLS || mode == DSS_VIT_RAGGED_PAD,
              "vit_ragged: unknown mode %d", mode);
  DSS_REQUIRE(n_out >= 0, "vit_ragged: negative n_max %d", n_out);
  const dss_vit_config& c = h->cfg;
  const int P = c.patch;
  const bool pad = mode == DSS_VIT_RAGGED_PAD;
  long long px = 0, np = 0, M = 0, tiles = 0;
  for (int b = 0; b < B; ++b) {
    const int H = dims[2 * b], W = dims[2 * b + 1];
    DSS_REQUIRE(H >= 0 && W >= 0, "vit_ragged: image %d has negative size %dx%d", b, H, W);
    if (pad)
      DSS_REQUIRE(H > 0 && W > 0, "vit_ragged: image %d (%dx%d) has no pixels", b, H, W);
    else
      DSS_REQUIRE(H >= P && W >= P, "vit_ragged: image %d (%dx%d) is smaller than one %d-pixel patch", b, H, W, P);
    const long long Hp = pad ? cdiv(H, P) : H / P, Wp = pad ? cdiv(W, P) : W / P;
    DSS_REQUIRE(!n_out || Hp * Wp <= n_out, "vit_ragged: image %d (%dx%d) has %lld patches, more than n_max = %d", b, H,
                W, Hp * Wp, n_out);
    px += (long long)H * W;
    np += Hp * Wp;
    M += Hp * Wp + 1;
    tiles += (Hp * Wp + RAGGED_TILE) / RAGGED_TILE;
  }
  // row counts are the extents of the tensor maps and GEMM problems (int); tile counts a grid dimension; a padded
  // output's rows are int table entries
  if (M > INT_MAX - 2 * RAGGED_TILE || tiles > INT_MAX || (long long)B * n_out > INT_MAX) {
    set_error("vit_ragged: %lld token rows (%lld output rows) do not fit the tensor-map extents", M,
              (long long)B * n_out);
    return DSS_ERR_UNSUPPORTED;
  }
  pl.n_patches = np;
  pl.M = M;
  size_t off = 0;
  auto part = [&off](size_t bytes) { const size_t o = off; off += align_up(bytes, 16); return o; };
  pl.t_imgs = part((size_t)B * sizeof(RaggedImage));
  pl.t_tiles = part((size_t)(B + 1) * 4);
  pl.t_prows = part((size_t)np * 4);
  pl.t_krows = part((size_t)M * 4);
  pl.tables_bytes = off;
  pl.vit_bytes = carve(c, (size_t)np, (size_t)M, (size_t)M, nullptr, h->precision).total;
  pl.total = pl.vit_bytes + align_up(pl.tables_bytes, 1024);
  if (!tables) return DSS_OK;

  pl.imgs.resize(B);
  pl.tile_prefix.assign(1, 0);
  pl.patch_rows.resize((size_t)np);
  pl.k_rows.resize((size_t)M);
  long long pxo = 0, po = 0, to = 0, fo = 0;
  for (int b = 0; b < B; ++b) {
    const int H = dims[2 * b], W = dims[2 * b + 1], Hp = pad ? cdiv(H, P) : H / P, Wp = pad ? cdiv(W, P) : W / P;
    const int Np = Hp * Wp;
    if (n_out) fo = (long long)b * n_out;
    RaggedImage& im = pl.imgs[b];
    im.px_off = pxo;
    im.H = H; im.W = W; im.Hp = Hp; im.Wp = Wp;
    im.patch_off = (int)po;
    im.tok_off = (int)to;
    im.stored = image_pos_is_stored(c.grid0, H, W, Hp, Wp, mode == DSS_VIT_RAGGED_CLS) ? 1 : 0;
    pl.tile_prefix.push_back(pl.tile_prefix.back() + (Np + RAGGED_TILE) / RAGGED_TILE);
    pl.k_rows[(size_t)to] = -1;
    for (int n = 0; n < Np; ++n) {
      pl.patch_rows[(size_t)(po + n)] = (int)(to + 1 + n);
      pl.k_rows[(size_t)(to + 1 + n)] = (int)(fo + n);
    }
    pxo += (long long)H * W;
    po += Np;
    to += Np + 1;
    fo += Np;
  }
  return DSS_OK;
}

// Validates a ragged batch (rmode: DSS_VIT_RAGGED_*, n_out: as ragged_plan) and uploads its tables into the workspace.
static int ragged_setup(dss_vit* h, const int* dims, int B, int rmode, int n_out, void* ws, size_t ws_bytes,
                        cudaStream_t st, RaggedPlan& pl, Ragged& rg) {
  int rc = ragged_plan(h, dims, B, rmode, n_out, true, pl);
  if (rc) return rc;
  DSS_REQUIRE(ws, "vit_ragged: null workspace");
  DSS_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "vit_ragged: workspace must be 256-byte aligned");
  DSS_REQUIRE(ws_bytes >= pl.total, "vit_ragged: workspace too small (%zu < %zu)", ws_bytes, pl.total);
  DSS_REQUIRE(h->loaded, "vit: weights not loaded");

  std::vector<uint8_t> blob(pl.tables_bytes);
  auto put = [&blob](size_t o, const void* src, size_t bytes) { if (bytes) std::memcpy(blob.data() + o, src, bytes); };
  put(pl.t_imgs, pl.imgs.data(), pl.imgs.size() * sizeof(RaggedImage));
  put(pl.t_tiles, pl.tile_prefix.data(), pl.tile_prefix.size() * 4);
  put(pl.t_prows, pl.patch_rows.data(), pl.patch_rows.size() * 4);
  put(pl.t_krows, pl.k_rows.data(), pl.k_rows.size() * 4);
  uint8_t* tb = reinterpret_cast<uint8_t*>(ws) + pl.vit_bytes;
  // pageable source: the call returns once the bytes are staged, so `blob` may go out of scope (no stream sync)
  DSS_CHECK_CUDA(cudaMemcpyAsync(tb, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
  rg.B = B;
  rg.n_patches = pl.n_patches;
  rg.M = pl.M;
  rg.tiles = pl.tile_prefix.back();
  rg.imgs = reinterpret_cast<const RaggedImage*>(tb + pl.t_imgs);
  rg.tile_prefix = reinterpret_cast<const int*>(tb + pl.t_tiles);
  rg.patch_rows = reinterpret_cast<const int*>(tb + pl.t_prows);
  rg.k_rows = reinterpret_cast<const int*>(tb + pl.t_krows);
  rg.n_out = n_out;
  return DSS_OK;
}

// n_full / mode as vit_run (0: K projection of block n_full, 2: final-norm CLS)
static int vit_ragged(dss_vit* h, const uint8_t* img, const int* dims, int B, int n_full, int mode, float* out, void* ws,
                      size_t ws_bytes, cudaStream_t st) {
  DSS_REQUIRE(img && out, "vit_ragged: null pointer");
  RaggedPlan pl;
  Ragged rg;
  int rc = ragged_setup(h, dims, B, mode == 0 ? DSS_VIT_RAGGED_K : DSS_VIT_RAGGED_CLS, 0, ws, ws_bytes, st, pl, rg);
  if (rc) return rc;
  return vit_run(h, img, B, 0, 0, n_full, mode, out, ws, pl.vit_bytes, st, 0, 1, nullptr, &rg);
}

}  // namespace dss

using namespace dss;

extern "C" int dss_vit_create(const dss_vit_config* cfg, dss_vit_t** out) {
  DSS_REQUIRE(cfg && out, "vit_create: null pointer");
  DSS_REQUIRE(cfg->dim == 384 || cfg->dim == 768, "vit_create: dim must be 384 or 768 (got %d)", cfg->dim);
  DSS_REQUIRE(cfg->heads > 0 && cfg->dim == cfg->heads * 64, "vit_create: head dim must be 64 (dim=%d heads=%d)",
              cfg->dim, cfg->heads);
  DSS_REQUIRE(cfg->patch == 8 || cfg->patch == 16, "vit_create: patch must be 8 or 16 (got %d)", cfg->patch);
  DSS_REQUIRE(cfg->depth > 0 && cfg->mlp_ratio > 0 && cfg->grid0 > 0, "vit_create: bad depth/mlp_ratio/grid0");
  dss_vit* h = new dss_vit();
  h->cfg = *cfg;
  *out = h;
  return DSS_OK;
}

extern "C" void dss_vit_destroy(dss_vit_t* h) {
  if (!h) return;
  if (h->arena) cudaFree(h->arena);
  delete h;
}

extern "C" int dss_vit_set_precision(dss_vit_t* h, int precision) {
  DSS_REQUIRE(h, "vit_set_precision: null handle");
  DSS_REQUIRE(precision == DSS_VIT_PRECISION_FP16 || precision == DSS_VIT_PRECISION_FP32,
              "vit_set_precision: precision must be DSS_VIT_PRECISION_FP16 (0) or DSS_VIT_PRECISION_FP32 (1), got %d",
              precision);
  DSS_REQUIRE(!h->arena, "vit_set_precision: the weights are already packed for precision %d; set the precision "
              "before dss_vit_load_weights", h->precision);
  h->precision = precision;
  return DSS_OK;
}

extern "C" int dss_vit_load_weights(dss_vit_t* h, const dss_vit_weights* w, dss_stream_t stream) {
  DSS_REQUIRE(h && w && w->blocks, "vit_load_weights: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dss_vit_config& c = h->cfg;
  const size_t d = c.dim, P = c.patch, hid = (size_t)c.mlp_ratio * d, Kp = 3 * P * P;
  // split weights (DSS_VIT_PRECISION_FP32): every row [hi | 64 lo | hi/64], three times as wide
  const size_t ks = h->precision == DSS_VIT_PRECISION_FP32 ? 3 : 1;
  // arena layout: f16 weights first (1 KB aligned for TMA), then fp32 vectors
  size_t off = 0;
  auto reserve = [&](size_t bytes) {
    size_t o = off;
    off += align_up(bytes, 1024);
    return o;
  };
  const size_t o_patch_w = reserve(d * Kp * 2 * ks), o_patch_b = reserve(d * 4), o_cls = reserve(d * 4);
  const size_t o_norm_w = reserve(d * 4), o_norm_b = reserve(d * 4);
  const size_t npos = ((size_t)c.grid0 * c.grid0 + 1) * d, o_pos = reserve(npos * 4);
  struct Off { size_t qkv_w, proj_w, fc1_w, fc2_w, ln1_w, ln1_b, ln2_w, ln2_b, qkv_b, proj_b, fc1_b, fc2_b; };
  std::vector<Off> bo(c.depth);
  for (int l = 0; l < c.depth; ++l) {
    bo[l].qkv_w = reserve(3 * d * d * 2 * ks); bo[l].proj_w = reserve(d * d * 2 * ks);
    bo[l].fc1_w = reserve(hid * d * 2 * ks); bo[l].fc2_w = reserve(d * hid * 2 * ks);
    bo[l].ln1_w = reserve(d * 4); bo[l].ln1_b = reserve(d * 4); bo[l].ln2_w = reserve(d * 4); bo[l].ln2_b = reserve(d * 4);
    bo[l].qkv_b = reserve(3 * d * 4); bo[l].proj_b = reserve(d * 4); bo[l].fc1_b = reserve(hid * 4); bo[l].fc2_b = reserve(d * 4);
  }
  if (h->arena && h->arena_bytes < off) { cudaFree(h->arena); h->arena = nullptr; }
  if (!h->arena) {
    DSS_CHECK_CUDA(cudaMalloc(&h->arena, off));
    h->arena_bytes = off;
  }
  uint8_t* base = reinterpret_cast<uint8_t*>(h->arena);
  // weight [rows, n / rows] fp32 -> fp16 operand at offset o
  auto cvt = [&](const float* src, size_t o, size_t n, size_t rows) -> int {
    DSS_REQUIRE(src, "vit_load_weights: null weight pointer");
    if (ks == 3) return launch_split_rows(src, base + o, (long long)rows, (int)(n / rows), 1, st, KC_MISC);
    LaunchScope scope(st, KC_MISC);
    f32_to_f16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, reinterpret_cast<__half*>(base + o), n);
    DSS_CHECK_CUDA(cudaGetLastError());
    return DSS_OK;
  };
  auto cpy = [&](const float* src, size_t o, size_t n) -> int {
    DSS_REQUIRE(src, "vit_load_weights: null weight pointer");
    DSS_CHECK_CUDA(cudaMemcpyAsync(base + o, src, n * 4, cudaMemcpyDeviceToDevice, st));
    return DSS_OK;
  };
  int rc;
  if ((rc = cvt(w->patch_w, o_patch_w, d * Kp, d))) return rc;
  if ((rc = cpy(w->patch_b, o_patch_b, d))) return rc;
  if ((rc = cpy(w->cls_token, o_cls, d))) return rc;
  DSS_REQUIRE(w->pos_embed, "vit_load_weights: null pos_embed");
  if ((rc = cpy(w->pos_embed, o_pos, npos))) return rc;
  h->pos_dev = reinterpret_cast<float*>(base + o_pos);
  h->patch_w = reinterpret_cast<__half*>(base + o_patch_w);
  h->patch_b = reinterpret_cast<float*>(base + o_patch_b);
  h->cls = reinterpret_cast<float*>(base + o_cls);
  h->norm_w = h->norm_b = nullptr;
  if (w->norm_w && w->norm_b) {
    if ((rc = cpy(w->norm_w, o_norm_w, d))) return rc;
    if ((rc = cpy(w->norm_b, o_norm_b, d))) return rc;
    h->norm_w = reinterpret_cast<float*>(base + o_norm_w);
    h->norm_b = reinterpret_cast<float*>(base + o_norm_b);
  }
  if ((rc = make_tmap_f16(&h->tm_patch, h->patch_w, (int)d, (int)(Kp * ks), 128 / 2))) return rc;
  h->blocks.resize(c.depth);
  for (int l = 0; l < c.depth; ++l) {
    const dss_vit_block_weights& s = w->blocks[l];
    BlockW& b = h->blocks[l];
    if ((rc = cvt(s.qkv_w, bo[l].qkv_w, 3 * d * d, 3 * d))) return rc;
    if ((rc = cvt(s.proj_w, bo[l].proj_w, d * d, d))) return rc;
    if ((rc = cvt(s.fc1_w, bo[l].fc1_w, hid * d, hid))) return rc;
    if ((rc = cvt(s.fc2_w, bo[l].fc2_w, d * hid, d))) return rc;
    if ((rc = cpy(s.ln1_w, bo[l].ln1_w, d))) return rc;
    if ((rc = cpy(s.ln1_b, bo[l].ln1_b, d))) return rc;
    if ((rc = cpy(s.ln2_w, bo[l].ln2_w, d))) return rc;
    if ((rc = cpy(s.ln2_b, bo[l].ln2_b, d))) return rc;
    if ((rc = cpy(s.qkv_b, bo[l].qkv_b, 3 * d))) return rc;
    if ((rc = cpy(s.proj_b, bo[l].proj_b, d))) return rc;
    if ((rc = cpy(s.fc1_b, bo[l].fc1_b, hid))) return rc;
    if ((rc = cpy(s.fc2_b, bo[l].fc2_b, d))) return rc;
    b.qkv_w = reinterpret_cast<__half*>(base + bo[l].qkv_w);
    b.proj_w = reinterpret_cast<__half*>(base + bo[l].proj_w);
    b.fc1_w = reinterpret_cast<__half*>(base + bo[l].fc1_w);
    b.fc2_w = reinterpret_cast<__half*>(base + bo[l].fc2_w);
    b.ln1_w = reinterpret_cast<float*>(base + bo[l].ln1_w); b.ln1_b = reinterpret_cast<float*>(base + bo[l].ln1_b);
    b.ln2_w = reinterpret_cast<float*>(base + bo[l].ln2_w); b.ln2_b = reinterpret_cast<float*>(base + bo[l].ln2_b);
    b.qkv_b = reinterpret_cast<float*>(base + bo[l].qkv_b); b.proj_b = reinterpret_cast<float*>(base + bo[l].proj_b);
    b.fc1_b = reinterpret_cast<float*>(base + bo[l].fc1_b); b.fc2_b = reinterpret_cast<float*>(base + bo[l].fc2_b);
    const int kd = (int)(d * ks), khid = (int)(hid * ks);   // row widths of the packed weights
    if ((rc = make_tmap_f16(&b.tm_qkv, b.qkv_w, (int)(3 * d), kd, gemm_tile_n() / 2))) return rc;
    if ((rc = make_tmap_f16(&b.tm_k, b.qkv_w + d * kd, (int)d, kd, 128 / 2))) return rc;
    if ((rc = make_tmap_f16(&b.tm_q, b.qkv_w, (int)d, kd, 128 / 2))) return rc;
    if ((rc = make_tmap_f16(&b.tm_v, b.qkv_w + 2 * d * kd, (int)d, kd, 128 / 2))) return rc;
    if ((rc = make_tmap_f16(&b.tm_proj, b.proj_w, (int)d, kd, gemm_tile_n() / 2))) return rc;
    if ((rc = make_tmap_f16(&b.tm_fc1, b.fc1_w, (int)hid, kd, gemm_tile_n() / 2))) return rc;
    if ((rc = make_tmap_f16(&b.tm_fc2, b.fc2_w, (int)d, khid, gemm_tile_n() / 2))) return rc;
  }
  h->loaded = true;
  return DSS_OK;
}

extern "C" size_t dss_vit_workspace_bytes(const dss_vit_t* h, int B, int H, int W) {
  if (!h || B <= 0 || H < h->cfg.patch || W < h->cfg.patch) return 0;
  const size_t Np = (size_t)(H / h->cfg.patch) * (W / h->cfg.patch);
  return carve(h->cfg, (size_t)B * Np, (size_t)B * (Np + 1), Np + 1, nullptr, h->precision).total;
}

extern "C" size_t dss_vit_forward_last_workspace_bytes(const dss_vit_t* h, int B, int H, int W, int pad) {
  if (!h || B <= 0 || H <= 0 || W <= 0) return 0;
  const int P = h->cfg.patch;
  if (!pad) return dss_vit_workspace_bytes(h, B, H, W);
  const size_t Np = (size_t)cdiv(H, P) * cdiv(W, P);
  return carve(h->cfg, (size_t)B * Np, (size_t)B * (Np + 1), Np + 1, nullptr, h->precision).total;
}

extern "C" int dss_vit_forward_last(dss_vit_t* h, const uint8_t* images_u8, int B, int H, int W, int pad, int which,
                                    float* feats_out, float* cls_attn_out, void* ws, size_t ws_bytes,
                                    dss_stream_t stream) {
  DSS_REQUIRE(h, "vit_forward_last: null handle");
  DSS_REQUIRE(which >= 0 && which <= 2, "vit_forward_last: which must be 0 (q), 1 (k) or 2 (v), got %d", which);
  DSS_REQUIRE(feats_out || cls_attn_out, "vit_forward_last: null pointer (no output requested)");
  DSS_REQUIRE(B > 0 && H > 0 && W > 0, "vit_forward_last: empty image batch");
  return vit_run(h, images_u8, B, H, W, h->cfg.depth - 1, 3, feats_out, ws, ws_bytes, static_cast<cudaStream_t>(stream),
                 pad, which, cls_attn_out);
}

extern "C" int dss_vit_forward_k(dss_vit_t* h, const uint8_t* images_u8, int B, int H, int W, int which_block,
                                 float* k_out, void* ws, size_t ws_bytes, dss_stream_t stream) {
  DSS_REQUIRE(h, "vit_forward_k: null handle");
  const int depth = h->cfg.depth;
  DSS_REQUIRE(which_block >= -depth && which_block < depth, "vit_forward_k: which_block %d out of range", which_block);
  const int blk = which_block < 0 ? which_block + depth : which_block;
  return vit_run(h, images_u8, B, H, W, blk, 0, k_out, ws, ws_bytes, static_cast<cudaStream_t>(stream));
}

extern "C" int dss_vit_forward_tokens(dss_vit_t* h, const uint8_t* images_u8, int B, int H, int W, int n_blocks,
                                      float* x_out, void* ws, size_t ws_bytes, dss_stream_t stream) {
  DSS_REQUIRE(h, "vit_forward_tokens: null handle");
  DSS_REQUIRE(n_blocks >= 0 && n_blocks <= h->cfg.depth, "vit_forward_tokens: n_blocks %d out of range", n_blocks);
  return vit_run(h, images_u8, B, H, W, n_blocks, 1, x_out, ws, ws_bytes, static_cast<cudaStream_t>(stream));
}

extern "C" int dss_vit_forward_cls(dss_vit_t* h, const uint8_t* images_u8, int B, int H, int W, float* cls_out, void* ws,
                                   size_t ws_bytes, dss_stream_t stream) {
  DSS_REQUIRE(h, "vit_forward_cls: null handle");
  return vit_run(h, images_u8, B, H, W, h->cfg.depth, 2, cls_out, ws, ws_bytes, static_cast<cudaStream_t>(stream));
}

extern "C" size_t dss_vit_ragged_workspace_bytes(const dss_vit_t* h, const int* dims_host, int B, int mode) {
  RaggedPlan pl;
  return ragged_plan(h, dims_host, B, mode, 0, false, pl) == DSS_OK ? pl.total : 0;
}

extern "C" int dss_vit_forward_k_ragged(dss_vit_t* h, const uint8_t* images_u8, const int* dims_host, int B,
                                        int which_block, float* k_out, void* ws, size_t ws_bytes, dss_stream_t stream) {
  DSS_REQUIRE(h, "vit_forward_k_ragged: null handle");
  const int depth = h->cfg.depth;
  DSS_REQUIRE(which_block >= -depth && which_block < depth, "vit_forward_k_ragged: which_block %d out of range",
              which_block);
  const int blk = which_block < 0 ? which_block + depth : which_block;
  return vit_ragged(h, images_u8, dims_host, B, blk, 0, k_out, ws, ws_bytes, static_cast<cudaStream_t>(stream));
}

extern "C" int dss_vit_forward_cls_ragged(dss_vit_t* h, const uint8_t* images_u8, const int* dims_host, int B,
                                          float* cls_out, void* ws, size_t ws_bytes, dss_stream_t stream) {
  DSS_REQUIRE(h, "vit_forward_cls_ragged: null handle");
  return vit_ragged(h, images_u8, dims_host, B, h->cfg.depth, 2, cls_out, ws, ws_bytes,
                    static_cast<cudaStream_t>(stream));
}

extern "C" int dss_vit_forward_last_ragged(dss_vit_t* h, const uint8_t* images_u8, const int* dims_host, int B,
                                           int pad, int which, float* feats_out, int n_max, float* cls_attn_out,
                                           void* ws, size_t ws_bytes, dss_stream_t stream) {
  DSS_REQUIRE(h, "vit_forward_last_ragged: null handle");
  DSS_REQUIRE(pad == 0 || pad == 1, "vit_forward_last_ragged: pad must be 0 or 1, got %d", pad);
  DSS_REQUIRE(which >= 0 && which <= 2, "vit_forward_last_ragged: which must be 0 (q), 1 (k) or 2 (v), got %d", which);
  DSS_REQUIRE(images_u8 && (feats_out || cls_attn_out), "vit_forward_last_ragged: null pointer");
  DSS_REQUIRE(n_max > 0, "vit_forward_last_ragged: n_max must be positive (got %d)", n_max);
  DSS_REQUIRE(!cls_attn_out || B <= 65535, "vit_forward_last_ragged: B = %d CLS attention rows exceed one grid column", B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RaggedPlan pl;
  Ragged rg;
  int rc = ragged_setup(h, dims_host, B, pad ? DSS_VIT_RAGGED_PAD : DSS_VIT_RAGGED_K, n_max, ws, ws_bytes, st, pl, rg);
  if (rc) return rc;
  return vit_run(h, images_u8, B, 0, 0, h->cfg.depth - 1, 3, feats_out, ws, pl.vit_bytes, st, pad, which,
                 cls_attn_out, &rg);
}

extern "C" int dss_vit_pos_embed_ragged(dss_vit_t* h, const int* dims_host, int B, int mode, float* pos_out, void* ws,
                                         size_t ws_bytes, dss_stream_t stream) {
  DSS_REQUIRE(h && pos_out, "vit_pos_embed_ragged: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RaggedPlan pl;
  Ragged rg;
  int rc = ragged_setup(h, dims_host, B, mode, 0, ws, ws_bytes, st, pl, rg);
  if (rc) return rc;
  // the forward's first step (it also writes the CLS rows of the workspace's residual stream)
  const VitWs w = carve(h->cfg, (size_t)pl.n_patches, (size_t)pl.M, (size_t)pl.M, ws, h->precision);
  if ((rc = launch_pos_cls(h, RaggedRows{rg.imgs, B}, B, pl.M, w, st))) return rc;
  DSS_CHECK_CUDA(cudaMemcpyAsync(pos_out, w.pos, (size_t)pl.M * h->cfg.dim * sizeof(float), cudaMemcpyDeviceToDevice,
                                 st));
  return DSS_OK;
}

extern "C" int dss_pos_embed_interp_host(const float* pos_embed_host, int grid0, int d, int Hp, int Wp,
                                         float* out_host) {
  DSS_REQUIRE(pos_embed_host && out_host && grid0 > 0 && d > 0 && Hp > 0 && Wp > 0, "pos_embed_interp_host: bad args");
  interp_pos_host(pos_embed_host, grid0, d, Hp, Wp, Hp == Wp, out_host);
  return DSS_OK;
}
