// Patch-affinity build: W = relu(F^ F^T) / max (+ lambda * colour counts)   (reference extract/extract.py:148,191-221)
//
// The Gram product runs on the tensor cores (wgmma) at fp32-equivalent accuracy. The eigenvectors of the graph
// Laplacian move by 2e-4..8e-4 when the features are merely rounded to bf16 (SURVEY 8a-4), so each normalised
// feature x is split as x = hi + lo with hi = fp16(x), lo = x - hi (|lo| <= 2^-12 |x|) and
//     x.y ~= hi.hi' + (hi/64).(64 lo') + (64 lo).(hi'/64)              (lo.lo' ~ 2^-24 is dropped)
// i.e. ONE fp16 GEMM with K = 3d over S = [hi | hi/64 | 64 lo] against the same array with the last two groups of
// K slabs swapped. The 2^+-6 factors keep every operand inside the fp16 normal range. The split itself is exact to
// ~2^-22 per product; the error that remains comes from the wgmma fp32 accumulation over 3 d / 16 k-steps. Measured
// max |W - W_float64| on an H100 80GB HBM3 at 400 W (normalised rows, d = 384): 5e-6, three times a plain fp32 product's 1.6e-6
// (d = 768: 9e-6 against 1e-6); DESIGN.md section 3, tests/test_affinity_exact_gpu.py.
// The GEMM itself is gemm.cu's TMA/wgmma kernel in batched mode with the affinity epilogue (relu, /max,
// + lambda*counts, zero padding of the row pitch) fused.
#include "common.cuh"

namespace dss {

// per-image max |f| (only needed when the features are NOT normalised: they are pre-scaled by a power of two so
// that fp16 cannot overflow; the scale cancels in W / max(W))
__global__ void __launch_bounds__(256)
absmax_kernel(const float* __restrict__ f, unsigned int* __restrict__ img_absmax, int rows, int N, int d) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* x = f + (long long)row * d;
  float m = 0.f;
  for (int k = lane; k < d; k += 32) m = fmaxf(m, fabsf(x[k]));
  m = warp_max(m);
  if (lane == 0) atomicMax(img_absmax + row / N, __float_as_uint(m));
}

// One warp per row: x^ = x / max(||x||, 1e-12) (F.normalize) or x * 2^-e; writes S[row] = [hi | hi/64 | 64 lo]
// (each group padded with zeros to dpad columns) and accumulates the per-image max of the Gram diagonal
// (== max of the whole matrix by Cauchy-Schwarz) with an integer atomicMax on the float bits.
__global__ void __launch_bounds__(256)
rownorm_split_kernel(const float* __restrict__ f, __half* __restrict__ S, unsigned int* __restrict__ img_max,
                     const unsigned int* __restrict__ img_absmax, int rows, int N, int d, int dpad, int normalize) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* x = f + (long long)row * d;
  __half* s = S + (long long)row * 3 * dpad;
  float ss = 0.f;
  for (int k = lane; k < d; k += 32) ss = fmaf(x[k], x[k], ss);
  ss = warp_sum(ss);
  const float denom = fmaxf(sqrtf(ss), 1e-12f);
  float pre = 1.0f;
  if (!normalize) {
    const float am = __uint_as_float(img_absmax[row / N]);
    if (am > 0.f) pre = exp2f(-ceilf(log2f(am)));
  }
  float s2 = 0.f;
  for (int k = lane; k < dpad; k += 32) {
    float v = 0.f;
    if (k < d) v = normalize ? x[k] / denom : x[k] * pre;
    store_split(s + k, dpad, 0, v);
    s2 = fmaf(v, v, s2);
  }
  s2 = warp_sum(s2);
  if (lane == 0) atomicMax(img_max + row / N, __float_as_uint(fmaxf(s2, 0.f)));
}

// F.normalize(p=2, dim=-1): one warp per row
__global__ void __launch_bounds__(256)
normalize_rows_kernel(const float* __restrict__ f, float* __restrict__ out, int rows, int d) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* x = f + (long long)row * d;
  float ss = 0.f;
  for (int k = lane; k < d; k += 32) ss = fmaf(x[k], x[k], ss);
  const float denom = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
  for (int k = lane; k < d; k += 32) out[(long long)row * d + k] = x[k] / denom;
}

// F.interpolate(mode='bilinear', align_corners=False) on a [Hp, Wp] grid of d-channel features stored [N, d]
__global__ void __launch_bounds__(256)
upsample_bilinear_kernel(const float* __restrict__ f, float* __restrict__ out, int Hp, int Wp, int d, int Hl, int Wl) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x;  // output pixel
  const int oy = pix / Wl, ox = pix % Wl;
  const float sy = fmaxf(((float)oy + 0.5f) * ((float)Hp / (float)Hl) - 0.5f, 0.f);
  const float sx = fmaxf(((float)ox + 0.5f) * ((float)Wp / (float)Wl) - 0.5f, 0.f);
  const int y0 = (int)sy, x0 = (int)sx;
  const int y1 = y0 + (y0 < Hp - 1 ? 1 : 0), x1 = x0 + (x0 < Wp - 1 ? 1 : 0);
  const float ly = sy - (float)y0, lx = sx - (float)x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const float* base = f + (long long)b * Hp * Wp * d;
  const float* p00 = base + (long long)(y0 * Wp + x0) * d;
  const float* p01 = base + (long long)(y0 * Wp + x1) * d;
  const float* p10 = base + (long long)(y1 * Wp + x0) * d;
  const float* p11 = base + (long long)(y1 * Wp + x1) * d;
  float* o = out + ((long long)b * Hl * Wl + pix) * d;
  for (int c = threadIdx.x; c < d; c += blockDim.x)
    o[c] = hy * (hx * p00[c] + lx * p01[c]) + ly * (hx * p10[c] + lx * p11[c]);
}

// D = W 1 from the per-tile partial sums of the symmetric affinity epilogue (gemm.cu), in a fixed order: row m of
// row tile I receives the row sums of tiles (I, j >= I) [slots 4 j + slice] and the column sums of tiles (i < I, I)
// [slots 4 tiles + 4 i + lane quarter].
__global__ void __launch_bounds__(256)
degree_reduce_kernel(const float* __restrict__ part, float* __restrict__ deg, int N, int tiles, int ld_part) {
  const int z = blockIdx.y;
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= N) return;
  const float* p = part + (long long)z * (8 * tiles) * ld_part + m;
  const int I = m >> 7;
  float s = 0.f;
  for (int k = 4 * I; k < 4 * tiles; ++k) s += p[(long long)k * ld_part];
  for (int k = 0; k < 4 * I; ++k) s += p[(long long)(4 * tiles + k) * ld_part];
  deg[(long long)z * N + m] = s;
}

static size_t degpart_bytes(int B, int N) {
  const int tiles = (N + 127) / 128;
  return align_up((size_t)B * 8 * tiles * (tiles * 128) * sizeof(float), 1024);
}

static size_t split_bytes(int B, int N, int d) {
  const int dpad = (d + 63) / 64 * 64;
  return align_up((size_t)B * N * 3 * dpad * sizeof(__half) + 128 * 3 * dpad * sizeof(__half), 1024);  // + tile overrun
}

}  // namespace dss

using namespace dss;

extern "C" size_t dss_affinity_workspace_bytes(int B, int N, int d) {
  if (B <= 0 || N <= 0 || d <= 0) return 0;
  return split_bytes(B, N, d) + 2 * align_up((size_t)B * sizeof(unsigned int), 256) + degpart_bytes(B, N) +
         align_up((size_t)B * N * sizeof(float), 256);   // + degree output when the caller does not ask for it
}

namespace dss {
// dss_affinity; `trace` (if not null) selects the phase-traced GEMM (dss_debug_affinity_trace)
static int affinity_run(const float* feats, int B, int N, int d, int flags, const uint8_t* color_counts,
                        float color_lambda, float* Wmat, int ldw, float* degree, void* ws, size_t ws_bytes,
                        dss_stream_t stream, unsigned long long* trace, size_t trace_bytes) {
  DSS_REQUIRE(feats && Wmat && ws, "affinity: null pointer");
  DSS_REQUIRE(B > 0 && N > 0 && d > 0, "affinity: empty problem B=%d N=%d d=%d", B, N, d);
  DSS_REQUIRE(ldw >= N && ldw % 4 == 0, "affinity: ldw must be >= N and a multiple of 4 (N=%d ldw=%d)", N, ldw);
  DSS_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "affinity: workspace must be 256-byte aligned");
  DSS_REQUIRE((reinterpret_cast<uintptr_t>(Wmat) & 15) == 0, "affinity: W must be 16-byte aligned");
  if (ws_bytes < dss_affinity_workspace_bytes(B, N, d)) {
    set_error("affinity: workspace too small (%zu < %zu)", ws_bytes, dss_affinity_workspace_bytes(B, N, d));
    return DSS_ERR_WORKSPACE;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int dpad = (d + 63) / 64 * 64;
  const int normalize = (flags & DSS_AFF_NORMALIZE) ? 1 : 0;
  __half* S = reinterpret_cast<__half*>(ws);
  unsigned int* img_max = reinterpret_cast<unsigned int*>(reinterpret_cast<uint8_t*>(ws) + split_bytes(B, N, d));
  unsigned int* img_absmax = img_max + align_up((size_t)B * sizeof(unsigned int), 256) / sizeof(unsigned int);
  DSS_CHECK_CUDA(cudaMemsetAsync(img_max, 0, 2 * align_up((size_t)B * sizeof(unsigned int), 256), st));
  const int rows = B * N;
  if (!normalize) {
    LaunchScope scope(st, KC_ROWNORM);
    absmax_kernel<<<cdiv(rows, 8), 256, 0, st>>>(feats, img_absmax, rows, N, d);
    DSS_CHECK_CUDA(cudaGetLastError());
  }
  {
    LaunchScope scope(st, KC_ROWNORM);
    rownorm_split_kernel<<<cdiv(rows, 8), 256, 0, st>>>(feats, S, img_max, img_absmax, rows, N, d, dpad, normalize);
    DSS_CHECK_CUDA(cudaGetLastError());
  }
  CUtensorMap tmS, tmS_half;   // A operand: 128-row boxes; B operand: 64-row half boxes (multicast inside the CTA pair)
  int rc = make_tmap_f16(&tmS, S, rows, 3 * dpad, 128);
  if (rc) return rc;
  if ((rc = make_tmap_f16(&tmS_half, S, rows, 3 * dpad, 64))) return rc;
  const size_t flag_bytes = 2 * align_up((size_t)B * sizeof(unsigned int), 256);
  float* deg_part = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws) + split_bytes(B, N, d) + flag_bytes);
  float* deg_out = degree ? degree
                          : reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(deg_part) + degpart_bytes(B, N));
  const int tiles = (N + 127) / 128, ld_part = tiles * 128;
  // The GEMM covers the columns of the image's 128-wide tiles (fewer if the pitch ends sooner): the degree partial
  // slots are laid out by those tiles in the epilogue and in degree_reduce_kernel alike. A wider pitch is zeroed here.
  const int ncols = ldw < ld_part ? ldw : ld_part;
  if (ldw > ncols)
    DSS_CHECK_CUDA(cudaMemset2DAsync(Wmat + ncols, (size_t)ldw * sizeof(float), 0, (size_t)(ldw - ncols) * sizeof(float),
                                     (size_t)B * N, st));
  if ((rc = affinity_gemm_tc(tmS, tmS_half, B, N, dpad, Wmat, ldw, ncols, img_max, normalize ? nullptr : img_absmax,
                             color_counts, color_lambda,
                             ((flags & DSS_AFF_THRESHOLD_AT_ZERO) ? 1 : 0) | ((flags & DSS_AFF_NO_MAX_SCALE) ? 2 : 0),
                             deg_part, ld_part, st, trace, trace_bytes)))
    return rc;
  {
    LaunchScope scope(st, KC_ROWNORM);
    degree_reduce_kernel<<<dim3(cdiv(N, 256), B), 256, 0, st>>>(deg_part, deg_out, N, tiles, ld_part);
    DSS_CHECK_CUDA(cudaGetLastError());
  }
  return DSS_OK;
}
}  // namespace dss

extern "C" int dss_affinity(const float* feats, int B, int N, int d, int flags, const uint8_t* color_counts,
                            float color_lambda, float* Wmat, int ldw, float* degree, void* ws, size_t ws_bytes,
                            dss_stream_t stream) {
  return affinity_run(feats, B, N, d, flags, color_counts, color_lambda, Wmat, ldw, degree, ws, ws_bytes, stream,
                      nullptr, 0);
}

extern "C" int dss_debug_affinity_trace(const float* feats, int B, int N, int d, int flags, const uint8_t* color_counts,
                                        float color_lambda, float* Wmat, int ldw, float* degree, void* ws,
                                        size_t ws_bytes, unsigned long long* trace, size_t trace_bytes,
                                        dss_stream_t stream) {
  DSS_REQUIRE(trace != nullptr, "debug_affinity_trace: null trace");
  return affinity_run(feats, B, N, d, flags, color_counts, color_lambda, Wmat, ldw, degree, ws, ws_bytes, stream,
                      trace, trace_bytes);
}

extern "C" int dss_normalize_rows(const float* feats, int rows, int d, float* out, dss_stream_t stream) {
  DSS_REQUIRE(feats && out && rows > 0 && d > 0, "normalize_rows: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LaunchScope scope(st, KC_ROWNORM);
  normalize_rows_kernel<<<cdiv(rows, 8), 256, 0, st>>>(feats, out, rows, d);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

extern "C" int dss_upsample_bilinear(const float* feats, int B, int Hp, int Wp, int d, int Hl, int Wl, float* out,
                                     dss_stream_t stream) {
  DSS_REQUIRE(feats && out, "upsample: null pointer");
  DSS_REQUIRE(B > 0 && Hp > 0 && Wp > 0 && d > 0 && Hl > 0 && Wl > 0, "upsample: empty problem");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LaunchScope scope(st, KC_MISC);
  upsample_bilinear_kernel<<<dim3(Hl * Wl, B), 128, 0, st>>>(feats, out, Hp, Wp, d, Hl, Wl);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}
