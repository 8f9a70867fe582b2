// Device half of the reference's semantic-segmentation recipe (extract/extract.py:429-599):
//   dss_segment_bboxes : erode / dilate every segment of the multi-region label maps and take its bounding box
//                        (_extract_bbox, extract.py:429-470; skimage binary_erosion / binary_dilation with the 3x3 cross)
//   dss_covariance     : column mean and centred covariance of the box features, the covariance-eigh route of
//                        scikit-learn's PCA (extract.py:573-577); the eigenvectors come from dss_eigsh_topk
//   dss_pca_project    : Y = (X - mean) V^T
//   dss_kmeans         : k-means over the whole data set (extract.py:579-582; see include/dss_b200.h for how it relates
//                        to the reference's MiniBatchKMeans)
// Every reduction is bit-reproducible: floating-point partial sums are written to fixed per-CTA slots and combined in
// a fixed order, and the k-means centre sums are accumulated in 64-bit fixed point, whose addition is associative.
// The library does not synchronise: k-means enqueues max_iter iterations whose kernels return at once after a
// device-side flag says the run has stopped.
#include <limits.h>
#include <math.h>

#include "common.cuh"
#include "kmeans_common.cuh"

namespace dss {

// ================================================================================================ bounding boxes
constexpr int BB_THREADS = 256;
constexpr int BB_MAX_PIXELS = 128 * 128;

// one CTA per (image, label value): blockIdx.x = image * 256 + value
__global__ void __launch_bounds__(BB_THREADS)
segment_bbox_kernel(const uint8_t* __restrict__ maps, int H, int W, int num_erode, int num_dilate,
                    int* __restrict__ boxes, uint8_t* __restrict__ present) {
  extern __shared__ uint8_t bb_smem[];
  __shared__ int s_box[4];
  const int HW = H * W, tid = threadIdx.x;
  const int b = blockIdx.x >> 8, v = blockIdx.x & 255;
  const uint8_t* m = maps + (long long)b * HW;
  uint8_t* cur = bb_smem;
  uint8_t* nxt = bb_smem + HW;
  int any = 0;
  for (int i = tid; i < HW; i += BB_THREADS) {
    const uint8_t s = m[i] == v;
    cur[i] = s;
    any |= s;
  }
  const int here = __syncthreads_or(any);
  const long long o = (long long)b * 256 + v;
  if (tid == 0) present[o] = (uint8_t)(here != 0);
  if (!here) {
    if (tid < 4) boxes[o * 4 + tid] = 0;
    return;
  }
  // erosion: pixels outside the image count as set; dilation: as unset. A step whose result is empty is discarded
  // (extract_utils.py:115-121), so the mask is never empty.
  for (int r = 0; r < num_erode + num_dilate; ++r) {
    const bool erode = r < num_erode;
    int set = 0;
    for (int i = tid; i < HW; i += BB_THREADS) {
      const int y = i / W, x = i - y * W;
      bool s;
      if (erode)
        s = cur[i] && (y == 0 || cur[i - W]) && (y == H - 1 || cur[i + W]) && (x == 0 || cur[i - 1]) &&
            (x == W - 1 || cur[i + 1]);
      else
        s = cur[i] || (y > 0 && cur[i - W]) || (y < H - 1 && cur[i + W]) || (x > 0 && cur[i - 1]) ||
            (x < W - 1 && cur[i + 1]);
      nxt[i] = s;
      set |= s;
    }
    if (__syncthreads_or(set)) {   // block-uniform
      uint8_t* t = cur; cur = nxt; nxt = t;
    }
  }
  if (tid == 0) { s_box[0] = W; s_box[1] = H; s_box[2] = -1; s_box[3] = -1; }
  __syncthreads();
  int x0 = W, y0 = H, x1 = -1, y1 = -1;
  for (int i = tid; i < HW; i += BB_THREADS) {
    if (!cur[i]) continue;
    const int y = i / W, x = i - y * W;
    x0 = min(x0, x); y0 = min(y0, y); x1 = max(x1, x); y1 = max(y1, y);
  }
  atomicMin(&s_box[0], x0); atomicMin(&s_box[1], y0); atomicMax(&s_box[2], x1); atomicMax(&s_box[3], y1);
  __syncthreads();
  if (tid < 4) boxes[o * 4 + tid] = tid < 2 ? s_box[tid] : s_box[tid] + 1;   // [xmin, ymin, xmax + 1, ymax + 1]
}

// ================================================================================================ shared reductions
constexpr int CL_THREADS = 256;
constexpr int CL_WARPS = CL_THREADS / 32;

// block sum in a fixed order (lane 0 of each warp after a shfl_down tree, then the warps in order); all threads get it
template <int NT>
__device__ __forceinline__ double block_sum_fixed(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < NT / 32; ++i) s += red[i];
  return s;
}

// per-CTA column sums of x and x^2 (fp64) over a contiguous row range, and the largest |x| (order-free max)
__global__ void __launch_bounds__(CL_THREADS)
colstats_kernel(const float* __restrict__ X, int M, int d, int rows_per_cta, double* __restrict__ part,
                unsigned* __restrict__ maxabs_bits) {
  const int g = blockIdx.x;
  const int r0 = g * rows_per_cta, r1 = min(M, r0 + rows_per_cta);
  float amax = 0.f;
  for (int j = threadIdx.x; j < d; j += CL_THREADS) {
    double s = 0.0, s2 = 0.0;
    for (int r = r0; r < r1; ++r) {
      const float v = X[(long long)r * d + j];
      s += v;
      s2 += (double)v * v;
      amax = fmaxf(amax, fabsf(v));
    }
    part[((long long)g * d + j) * 2 + 0] = s;
    part[((long long)g * d + j) * 2 + 1] = s2;
  }
  amax = warp_max(amax);
  if ((threadIdx.x & 31) == 0) atomicMax(maxabs_bits, __float_as_uint(amax));   // non-negative floats order as uints
}

// ================================================================================================ covariance / PCA
constexpr int COV_TILE = 64;
constexpr int COV_ROWS = 32;

__global__ void __launch_bounds__(CL_THREADS)
column_mean_kernel(const double* __restrict__ part, int G, int M, int d, double* __restrict__ mean,
                   float* __restrict__ mean_out) {
  for (int j = threadIdx.x; j < d; j += CL_THREADS) {
    double s = 0.0;
    for (int g = 0; g < G; ++g) s += part[((long long)g * d + j) * 2];
    mean[j] = s / M;
    if (mean_out) mean_out[j] = (float)(s / M);
  }
}

__device__ __forceinline__ void cov_tile_coords(int t, int nt, int& ti, int& tj) {
  ti = 0;
  while (t >= nt - ti) { t -= nt - ti; ++ti; }
  tj = ti + t;
}

// one 64 x 64 tile (ti <= tj) of sum_r (x_r - mean)(x_r - mean)^T over the row range of split blockIdx.y, in fp64
__global__ void __launch_bounds__(CL_THREADS)
covariance_tile_kernel(const float* __restrict__ X, int M, int d, const double* __restrict__ mean, int rows_per_split,
                       double* __restrict__ part) {
  __shared__ double As[COV_ROWS][COV_TILE], Bs[COV_ROWS][COV_TILE];
  const int nt = (d + COV_TILE - 1) / COV_TILE;
  int ti, tj;
  cov_tile_coords(blockIdx.x, nt, ti, tj);
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int r0 = blockIdx.y * rows_per_split, r1 = min(M, r0 + rows_per_split);
  double acc[4][4] = {};
  for (int rb = r0; rb < r1; rb += COV_ROWS) {
    for (int e = tid; e < COV_ROWS * COV_TILE; e += CL_THREADS) {
      const int rr = e / COV_TILE, cc = e % COV_TILE, r = rb + rr;
      const int ci = ti * COV_TILE + cc, cj = tj * COV_TILE + cc;
      As[rr][cc] = (r < r1 && ci < d) ? (double)X[(long long)r * d + ci] - mean[ci] : 0.0;
      Bs[rr][cc] = (r < r1 && cj < d) ? (double)X[(long long)r * d + cj] - mean[cj] : 0.0;
    }
    __syncthreads();
#pragma unroll 4
    for (int rr = 0; rr < COV_ROWS; ++rr) {
      double a[4], bv[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) { a[q] = As[rr][ty * 4 + q]; bv[q] = Bs[rr][tx * 4 + q]; }
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[p][q] = fma(a[p], bv[q], acc[p][q]);
    }
    __syncthreads();
  }
  double* out = part + ((long long)blockIdx.y * gridDim.x + blockIdx.x) * COV_TILE * COV_TILE;
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 4; ++q) out[(ty * 4 + p) * COV_TILE + tx * 4 + q] = acc[p][q];
}

// splits combined in order, / (M - 1), written to both triangles of C [d, ldc]
__global__ void __launch_bounds__(CL_THREADS)
covariance_combine_kernel(const double* __restrict__ part, int splits, int M, int d, float* __restrict__ C, int ldc) {
  const int nt = (d + COV_TILE - 1) / COV_TILE;
  int ti, tj;
  cov_tile_coords(blockIdx.x, nt, ti, tj);
  for (int e = threadIdx.x; e < COV_TILE * COV_TILE; e += CL_THREADS) {
    const int i = ti * COV_TILE + e / COV_TILE, j = tj * COV_TILE + e % COV_TILE;
    if (i >= d || j >= d) continue;
    double s = 0.0;
    for (int sp = 0; sp < splits; ++sp) s += part[((long long)sp * gridDim.x + blockIdx.x) * COV_TILE * COV_TILE + e];
    const float v = (float)(s / (double)(M - 1));
    C[(long long)i * ldc + j] = v;
    C[(long long)j * ldc + i] = v;
  }
}

// Y [M, p] = (X - mean) V^T, V [p, d]; 64 rows per CTA, p <= 64
__global__ void __launch_bounds__(CL_THREADS)
pca_project_kernel(const float* __restrict__ X, int M, int d, const float* __restrict__ mean, const float* __restrict__ V,
                   int p, float* __restrict__ Y) {
  __shared__ float Xs[64][33], Vs[64][33];
  const int tid = threadIdx.x, r = tid >> 2, cq = tid & 3;
  const long long row0 = (long long)blockIdx.x * 64;
  float acc[16] = {};
  for (int k0 = 0; k0 < d; k0 += 32) {
    for (int e = tid; e < 64 * 32; e += CL_THREADS) {
      const int rr = e >> 5, kk = e & 31, k = k0 + kk;
      const long long row = row0 + rr;
      Xs[rr][kk] = (row < M && k < d) ? X[row * d + k] - mean[k] : 0.f;
      Vs[rr][kk] = (rr < p && k < d) ? V[(long long)rr * d + k] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < 32; ++kk) {
      const float xv = Xs[r][kk];
#pragma unroll
      for (int q = 0; q < 16; ++q) acc[q] = fmaf(xv, Vs[cq + 4 * q][kk], acc[q]);
    }
    __syncthreads();
  }
  const long long row = row0 + r;
  if (row < M)
#pragma unroll
    for (int q = 0; q < 16; ++q)
      if (cq + 4 * q < p) Y[row * p + cq + 4 * q] = acc[q];
}

// ================================================================================================ k-means
constexpr int KM_CHUNK = 512;        // points per CTA of the point-parallel kernels (and per slot of the D^2 scan)
constexpr int KM_MAX_TRIALS = 8;
constexpr int KM_ACC_SLOTS = 64;     // point ranges of the centre accumulation

struct KmState {
  int done, strict, converged, iters, changed, pad;
  double tol_abs, scale;
  int cand[KM_MAX_TRIALS];
};

struct KmParams {
  const float* X;
  int M, dims, k, trials, max_iter;
  float tol;
  uint32_t seed;
  KmState* st;
  double* colpart;       // [Gc, dims, 2]
  unsigned* maxabs;      // [1]
  int Gc, rows_c;
  float* mind2;          // [M] squared distance to the closest centre
  double* chunksum;      // [G] sum of mind2 over each KM_CHUNK range
  double* potpart;       // [G, KM_MAX_TRIALS]
  double* inpart;        // [G]
  int G;
  long long* accs;       // [Gp, k, dims] fixed-point centre sums per point range
  int* cnts;             // [Gp, k]
  long long* tot;        // [k, dims]
  int* cnt;              // [k]
  int Gp, rows_p, DT;
  float* centers;        // [k, dims]
  int* labels;           // [M]
};

__device__ __forceinline__ long long km_fixed(float v, double scale) { return __double2ll_rn((double)v * scale); }

template <int NJ>
__device__ __forceinline__ void km_load_point(const float* __restrict__ x, int dims, int lane, float (&r)[NJ]) {
#pragma unroll
  for (int i = 0; i < NJ; ++i) {
    const int j = lane + 32 * i;
    r[i] = j < dims ? x[j] : 0.f;
  }
}
// squared distance of the warp's point (in registers, lane-strided) to c; a fixed-order tree, broadcast from lane 0
template <int NJ>
__device__ __forceinline__ float km_dist(const float (&r)[NJ], const float* __restrict__ c, int dims, int lane) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NJ; ++i) {
    const int j = lane + 32 * i;
    if (j < dims) { const float t = r[i] - c[j]; s = fmaf(t, t, s); }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  return __shfl_sync(0xffffffffu, s, 0);
}

// tolerance (sklearn _tolerance: tol * mean of the column variances) and the fixed-point scale: |x| < 2^e and
// M < 2^lm give |sum| < 2^62
__global__ void __launch_bounds__(CL_THREADS) km_prepare_kernel(KmParams p) {
  __shared__ double red[CL_WARPS];
  double vs = 0.0;
  for (int j = threadIdx.x; j < p.dims; j += CL_THREADS) {
    double s = 0.0, s2 = 0.0;
    for (int g = 0; g < p.Gc; ++g) {
      s += p.colpart[((long long)g * p.dims + j) * 2];
      s2 += p.colpart[((long long)g * p.dims + j) * 2 + 1];
    }
    const double mean = s / p.M;
    vs += s2 / p.M - mean * mean;
  }
  vs = block_sum_fixed<CL_THREADS>(vs, red);
  if (threadIdx.x == 0) {
    p.st->tol_abs = (double)p.tol * (vs / p.dims);
    const float amax = __uint_as_float(*p.maxabs);
    int e = 0;
    if (amax > 0.f) frexpf(amax, &e);
    int lm = 0;
    while ((1ll << lm) < (long long)p.M) ++lm;
    p.st->scale = ldexp(1.0, min(62 - e - lm, 900));
  }
}

// adds centre c: the first one uniformly at random, later ones the candidate with the smallest potential; then
// mind2 = min(mind2, distance to it) and the per-chunk sums of mind2 for the next D^2 draw
template <int NJ>
__global__ void __launch_bounds__(CL_THREADS) km_seed_update_kernel(KmParams p, int c) {
  __shared__ double red[CL_WARPS];
  __shared__ int s_best;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = blockIdx.x;
  if (tid == 0) {
    if (c == 0) {
      s_best = min(p.M - 1, (int)(seg_uniform(p.seed, 0u, 0u) * p.M));
    } else {
      int bt = 0;
      double bp = 0.0;
      for (int t = 0; t < p.trials; ++t) {
        double s = 0.0;
        for (int h = 0; h < p.G; ++h) s += p.potpart[(long long)h * KM_MAX_TRIALS + t];
        if (t == 0 || s < bp) { bp = s; bt = t; }
      }
      s_best = p.st->cand[bt];
    }
  }
  __syncthreads();
  const float* xb = p.X + (long long)s_best * p.dims;
  if (g == 0)
    for (int j = tid; j < p.dims; j += CL_THREADS) p.centers[(long long)c * p.dims + j] = xb[j];
  const int n0 = g * KM_CHUNK, n1 = min(p.M, n0 + KM_CHUNK);
  for (int n = n0 + warp; n < n1; n += CL_WARPS) {
    float r[NJ];
    km_load_point<NJ>(p.X + (long long)n * p.dims, p.dims, lane, r);
    const float d2 = km_dist<NJ>(r, xb, p.dims, lane);
    if (lane == 0) p.mind2[n] = c == 0 ? d2 : fminf(p.mind2[n], d2);
  }
  __syncthreads();
  double s = 0.0;
  for (int n = n0 + tid; n < n1; n += CL_THREADS) s += p.mind2[n];
  s = block_sum_fixed<CL_THREADS>(s, red);
  if (tid == 0) p.chunksum[g] = s;
}

// inclusive scan over KM_CHUNK threads in a fixed order (all threads of the block take part)
__device__ __forceinline__ double km_block_scan(double v, double* wsum) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  __syncthreads();
  if (lane == 31) wsum[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < KM_CHUNK / 32; ++w) wsum[w] += wsum[w - 1];
  __syncthreads();
  return warp > 0 ? v + wsum[warp - 1] : v;
}

// D^2 draws of the local trials of centre c: the candidate of a target u * pot is the first point whose inclusive
// prefix sum of mind2 exceeds it (first the chunk, from the chunk sums, then the point inside the chunk)
__global__ void __launch_bounds__(KM_CHUNK) km_seed_pick_kernel(KmParams p, int c) {
  __shared__ double wsum[KM_CHUNK / 32];
  __shared__ double tgt[KM_MAX_TRIALS], excl[KM_MAX_TRIALS];
  __shared__ int gsel[KM_MAX_TRIALS], nsel[KM_MAX_TRIALS];
  __shared__ double s_carry;
  const int tid = threadIdx.x;
  if (tid < KM_MAX_TRIALS) { gsel[tid] = INT_MAX; nsel[tid] = INT_MAX; }
  if (tid == 0) s_carry = 0.0;
  __syncthreads();
  for (int g0 = 0; g0 < p.G; g0 += KM_CHUNK) {
    const int g = g0 + tid;
    const double own = g < p.G ? p.chunksum[g] : 0.0;
    const double incl = s_carry + km_block_scan(own, wsum);
    __syncthreads();
    if (tid == KM_CHUNK - 1) s_carry = incl;
    __syncthreads();
  }
  const double pot = s_carry;   // the targets need the total: a first pass over the chunk sums
  __syncthreads();
  if (tid < p.trials) tgt[tid] = seg_uniform(p.seed, 0u, (uint32_t)(1 + (c - 1) * p.trials + tid)) * pot;
  if (tid == 0) s_carry = 0.0;
  __syncthreads();
  for (int g0 = 0; g0 < p.G; g0 += KM_CHUNK) {
    const int g = g0 + tid;
    const double own = g < p.G ? p.chunksum[g] : 0.0;
    const double incl = s_carry + km_block_scan(own, wsum);
    if (g < p.G)
      for (int t = 0; t < p.trials; ++t)
        if (incl > tgt[t]) atomicMin(&gsel[t], g);
    __syncthreads();
    if (g < p.G)
      for (int t = 0; t < p.trials; ++t)
        if (gsel[t] == g) excl[t] = incl - own;
    if (tid == KM_CHUNK - 1) s_carry = incl;
    __syncthreads();
  }
  for (int t = 0; t < p.trials; ++t) {
    const int g = gsel[t];   // block-uniform
    if (g == INT_MAX) {      // rounding put the target past the total: the last point, as a sequential walk would
      if (tid == 0) p.st->cand[t] = p.M - 1;
      continue;
    }
    const int n = g * KM_CHUNK + tid, nend = min(p.M, (g + 1) * KM_CHUNK);
    const double incl = km_block_scan(n < nend ? (double)p.mind2[n] : 0.0, wsum);
    if (n < nend && incl > tgt[t] - excl[t]) atomicMin(&nsel[t], n);
    __syncthreads();
    if (tid == 0) p.st->cand[t] = nsel[t] == INT_MAX ? nend - 1 : nsel[t];
  }
}

// potential sum_n min(mind2[n], |x_n - x_cand_t|^2) of every trial, per CTA
template <int NJ>
__global__ void __launch_bounds__(CL_THREADS) km_seed_pot_kernel(KmParams p) {
  __shared__ double wpart[CL_WARPS][KM_MAX_TRIALS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = blockIdx.x;
  double acc[KM_MAX_TRIALS] = {};
  const int n0 = g * KM_CHUNK, n1 = min(p.M, n0 + KM_CHUNK);
  for (int n = n0 + warp; n < n1; n += CL_WARPS) {
    float r[NJ];
    km_load_point<NJ>(p.X + (long long)n * p.dims, p.dims, lane, r);
    const float m = p.mind2[n];
    for (int t = 0; t < p.trials; ++t) {
      const float d2 = km_dist<NJ>(r, p.X + (long long)p.st->cand[t] * p.dims, p.dims, lane);
      acc[t] += fminf(m, d2);
    }
  }
  if (lane == 0)
    for (int t = 0; t < KM_MAX_TRIALS; ++t) wpart[warp][t] = acc[t];
  __syncthreads();
  if (tid < KM_MAX_TRIALS) {
    double s = 0.0;
    for (int w = 0; w < CL_WARPS; ++w) s += wpart[w][tid];
    p.potpart[(long long)g * KM_MAX_TRIALS + tid] = s;
  }
}

// E step: nearest centre (ties -> lower index), changed labels counted, per-CTA inertia.
// final_pass: the E step after the loop that makes the labels match the final centres (skipped when the labels
// already converged strictly).
template <int NJ>
__global__ void __launch_bounds__(CL_THREADS) km_assign_kernel(KmParams p, int final_pass) {
  extern __shared__ __align__(16) float km_cen[];
  __shared__ double red[CL_WARPS];
  __shared__ int s_changed;
  if (final_pass ? p.st->strict : p.st->done) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = blockIdx.x;
  for (int i = tid; i < p.k * p.dims; i += CL_THREADS) km_cen[i] = p.centers[i];
  if (tid == 0) s_changed = 0;
  __syncthreads();
  const int n0 = g * KM_CHUNK, n1 = min(p.M, n0 + KM_CHUNK);
  double inert = 0.0;
  int changed = 0;
  for (int n = n0 + warp; n < n1; n += CL_WARPS) {
    float r[NJ];
    km_load_point<NJ>(p.X + (long long)n * p.dims, p.dims, lane, r);
    float bd = INFINITY;
    int bc = 0;
    for (int c = 0; c < p.k; ++c) {
      const float d2 = km_dist<NJ>(r, km_cen + (long long)c * p.dims, p.dims, lane);
      if (d2 < bd) { bd = d2; bc = c; }
    }
    if (lane == 0) {
      changed += p.labels[n] != bc;
      p.labels[n] = bc;
      p.mind2[n] = bd;
      inert += bd;
    }
  }
  if (lane == 0 && changed) atomicAdd(&s_changed, changed);
  inert = block_sum_fixed<CL_THREADS>(inert, red);   // lane 0 of each warp holds the warp's points in order
  if (tid == 0) {
    p.inpart[g] = inert;
    if (s_changed) atomicAdd(&p.st->changed, s_changed);   // integer: order-free
  }
}

// M step, part 1: fixed-point sums of the points of each label over a point range and a column tile
__global__ void __launch_bounds__(CL_THREADS) km_accum_kernel(KmParams p) {
  extern __shared__ __align__(16) unsigned long long km_acc[];
  if (p.st->done || p.st->changed == 0) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = blockIdx.x;
  const int j0 = blockIdx.y * p.DT, dt = min(p.DT, p.dims - j0);
  int* cnt_s = reinterpret_cast<int*>(km_acc + (size_t)p.k * p.DT);
  for (int i = tid; i < p.k * dt; i += CL_THREADS) km_acc[i] = 0ull;
  for (int i = tid; i < p.k; i += CL_THREADS) cnt_s[i] = 0;
  __syncthreads();
  const double scale = p.st->scale;
  const int n0 = g * p.rows_p, n1 = min(p.M, n0 + p.rows_p);
  for (int n = n0 + warp; n < n1; n += CL_WARPS) {
    const int l = p.labels[n];
    const float* x = p.X + (long long)n * p.dims + j0;
    for (int jj = lane; jj < dt; jj += 32) atomicAdd(&km_acc[l * dt + jj], (unsigned long long)km_fixed(x[jj], scale));
    if (blockIdx.y == 0 && lane == 0) atomicAdd(&cnt_s[l], 1);
  }
  __syncthreads();
  for (int i = tid; i < p.k * dt; i += CL_THREADS) {
    const int c = i / dt, jj = i - c * dt;
    p.accs[((long long)g * p.k + c) * p.dims + j0 + jj] = (long long)km_acc[i];
  }
  if (blockIdx.y == 0)
    for (int i = tid; i < p.k; i += CL_THREADS) p.cnts[(long long)g * p.k + i] = cnt_s[i];
}

// M step, part 2: the point ranges combined
__global__ void __launch_bounds__(CL_THREADS) km_reduce_kernel(KmParams p) {
  if (p.st->done || p.st->changed == 0) return;
  const long long i = (long long)blockIdx.x * CL_THREADS + threadIdx.x;
  const long long kd = (long long)p.k * p.dims;
  if (i < kd) {
    long long s = 0;
    for (int g = 0; g < p.Gp; ++g) s += p.accs[(long long)g * kd + i];
    p.tot[i] = s;
  }
  if (i < p.k) {
    int s = 0;
    for (int g = 0; g < p.Gp; ++g) s += p.cnts[(long long)g * p.k + i];
    p.cnt[i] = s;
  }
}

// end of an iteration (one CTA): strict convergence, empty clusters re-seeded with the farthest points
// (sklearn _relocate_empty_clusters_dense), new centres, centre shift against the tolerance
constexpr int KM_FIN_THREADS = 1024;
__global__ void __launch_bounds__(KM_FIN_THREADS) km_finish_kernel(KmParams p) {
  __shared__ double red[KM_FIN_THREADS / 32];
  __shared__ float s_val[KM_FIN_THREADS / 32];
  __shared__ int s_idx[KM_FIN_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (p.st->done) return;
  const int it = p.st->iters + 1;
  const int changed = p.st->changed;
  __syncthreads();
  if (changed == 0) {   // labels did not change: converged, centres stay
    if (tid == 0) { p.st->done = 1; p.st->strict = 1; p.st->converged = 1; p.st->iters = it; }
    return;
  }
  const double scale = p.st->scale;
  for (int c = 0; c < p.k; ++c) {
    if (p.cnt[c] != 0) continue;   // block-uniform (global memory written by thread 0 before the last barrier)
    float bv = -INFINITY;
    int bi = 0;
    for (int n = tid; n < p.M; n += KM_FIN_THREADS) {
      const float v = p.mind2[n];
      if (v > bv) { bv = v; bi = n; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { s_val[warp] = bv; s_idx[warp] = bi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < KM_FIN_THREADS / 32; ++w)
        if (s_val[w] > s_val[0] || (s_val[w] == s_val[0] && s_idx[w] < s_idx[0])) { s_val[0] = s_val[w]; s_idx[0] = s_idx[w]; }
      const int far = s_idx[0], old = p.labels[far];
      const float* x = p.X + (long long)far * p.dims;
      for (int j = 0; j < p.dims; ++j) {
        const long long q = km_fixed(x[j], scale);
        p.tot[(long long)old * p.dims + j] -= q;
        p.tot[(long long)c * p.dims + j] = q;
      }
      p.cnt[old] -= 1;
      p.cnt[c] = 1;
      // the label stays the E step's (sklearn leaves it too): the next E step counts its changes against it
      p.mind2[far] = -1.f;   // not picked again for the next empty cluster
    }
    __syncthreads();
  }
  double shift = 0.0;
  for (int i = tid; i < p.k * p.dims; i += KM_FIN_THREADS) {
    const int c = i / p.dims;
    const float old = p.centers[i];
    const float nc = p.cnt[c] > 0 ? (float)((double)p.tot[i] / scale / (double)p.cnt[c]) : old;
    const double dl = (double)nc - (double)old;
    shift += dl * dl;
    p.centers[i] = nc;
  }
  shift = block_sum_fixed<KM_FIN_THREADS>(shift, red);
  if (tid == 0) {
    p.st->iters = it;
    p.st->changed = 0;
    if (shift <= p.st->tol_abs) { p.st->done = 1; p.st->converged = 1; }
    else if (it >= p.max_iter) p.st->done = 1;
  }
}

__global__ void __launch_bounds__(CL_THREADS) km_report_kernel(KmParams p, int* info, float* inertia) {
  __shared__ double red[CL_WARPS];
  double s = 0.0;
  for (int g = threadIdx.x; g < p.G; g += CL_THREADS) s += p.inpart[g];
  s = block_sum_fixed<CL_THREADS>(s, red);
  if (threadIdx.x == 0) {
    info[0] = p.st->iters;
    info[1] = p.st->converged;
    if (inertia) *inertia = (float)s;
  }
}

struct KmLayout {
  int G, Gc, rows_c, Gp, rows_p, DT;
  size_t off_colpart, off_maxabs, off_mind2, off_chunk, off_pot, off_inpart, off_accs, off_cnts, off_tot, off_cnt, total;
};

static KmLayout km_layout(int M, int dims, int k) {
  KmLayout L;
  L.G = cdiv(M, KM_CHUNK);
  L.Gc = M < 264 * 64 ? cdiv(M, 64) : 264;
  L.rows_c = cdiv(M, L.Gc);
  L.Gp = M < KM_ACC_SLOTS * 1024 ? cdiv(M, 1024) : KM_ACC_SLOTS;
  L.rows_p = cdiv(M, L.Gp);
  L.DT = dims < 8192 / k ? dims : 8192 / k;   // k * DT * 8 <= 64 KB of shared memory
  size_t o = align_up(sizeof(KmState), 256);
  L.off_colpart = o; o = align_up(o + (size_t)L.Gc * dims * 2 * 8, 256);
  L.off_maxabs = o;  o = align_up(o + 4, 256);
  L.off_mind2 = o;   o = align_up(o + (size_t)M * 4, 256);
  L.off_chunk = o;   o = align_up(o + (size_t)L.G * 8, 256);
  L.off_pot = o;     o = align_up(o + (size_t)L.G * KM_MAX_TRIALS * 8, 256);
  L.off_inpart = o;  o = align_up(o + (size_t)L.G * 8, 256);
  L.off_accs = o;    o = align_up(o + (size_t)L.Gp * k * dims * 8, 256);
  L.off_cnts = o;    o = align_up(o + (size_t)L.Gp * k * 4, 256);
  L.off_tot = o;     o = align_up(o + (size_t)k * dims * 8, 256);
  L.off_cnt = o;     o = align_up(o + (size_t)k * 4, 256);
  L.total = o;
  return L;
}

static bool km_supported(int dims, int k) { return (k <= 64 && dims <= 768) || (k <= 256 && dims <= 64); }

template <int NJ>
static int km_run(const KmParams& p, size_t cen_smem, size_t acc_smem, int nDT, cudaStream_t st, int* info,
                  float* inertia) {
  DSS_CHECK_CUDA(cudaFuncSetAttribute(km_assign_kernel<NJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cen_smem));
  DSS_CHECK_CUDA(cudaFuncSetAttribute(km_accum_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)acc_smem));
  {
    LaunchScope scope(st, KC_MISC);
    colstats_kernel<<<p.Gc, CL_THREADS, 0, st>>>(p.X, p.M, p.dims, p.rows_c, p.colpart, p.maxabs);
  }
  {
    LaunchScope scope(st, KC_MISC);
    km_prepare_kernel<<<1, CL_THREADS, 0, st>>>(p);
  }
  for (int c = 0; c < p.k; ++c) {
    if (c > 0) {
      { LaunchScope scope(st, KC_MISC); km_seed_pick_kernel<<<1, KM_CHUNK, 0, st>>>(p, c); }
      { LaunchScope scope(st, KC_MISC); km_seed_pot_kernel<NJ><<<p.G, CL_THREADS, 0, st>>>(p); }
    }
    LaunchScope scope(st, KC_MISC);
    km_seed_update_kernel<NJ><<<p.G, CL_THREADS, 0, st>>>(p, c);
  }
  DSS_CHECK_CUDA(cudaGetLastError());
  const unsigned red_grid = (unsigned)(((long long)p.k * p.dims + CL_THREADS - 1) / CL_THREADS);
  for (int it = 0; it < p.max_iter; ++it) {
    { LaunchScope scope(st, KC_MISC); km_assign_kernel<NJ><<<p.G, CL_THREADS, cen_smem, st>>>(p, 0); }
    { LaunchScope scope(st, KC_MISC); km_accum_kernel<<<dim3(p.Gp, nDT), CL_THREADS, acc_smem, st>>>(p); }
    { LaunchScope scope(st, KC_MISC); km_reduce_kernel<<<red_grid, CL_THREADS, 0, st>>>(p); }
    { LaunchScope scope(st, KC_MISC); km_finish_kernel<<<1, KM_FIN_THREADS, 0, st>>>(p); }
  }
  { LaunchScope scope(st, KC_MISC); km_assign_kernel<NJ><<<p.G, CL_THREADS, cen_smem, st>>>(p, 1); }
  { LaunchScope scope(st, KC_MISC); km_report_kernel<<<1, CL_THREADS, 0, st>>>(p, info, inertia); }
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

// ------------------------------------------------------------------------------------------ covariance workspace
struct CovLayout {
  int Gc, rows_c, nt, splits, rows_split;
  size_t off_maxabs, off_mean, off_part, total;
};

static CovLayout cov_layout(int M, int d) {
  CovLayout L;
  L.Gc = M < 264 * 64 ? cdiv(M, 64) : 264;
  L.rows_c = cdiv(M, L.Gc);
  const int nt1 = cdiv(d, COV_TILE);
  L.nt = nt1 * (nt1 + 1) / 2;
  L.splits = cdiv(264, L.nt);
  if (L.splits > cdiv(M, COV_ROWS)) L.splits = cdiv(M, COV_ROWS);
  L.rows_split = cdiv(cdiv(M, L.splits), COV_ROWS) * COV_ROWS;
  size_t o = align_up((size_t)L.Gc * d * 2 * 8, 256);
  L.off_maxabs = o; o = align_up(o + 4, 256);
  L.off_mean = o;   o = align_up(o + (size_t)d * 8, 256);
  L.off_part = o;   o = align_up(o + (size_t)L.splits * L.nt * COV_TILE * COV_TILE * 8, 256);
  L.total = o;
  return L;
}

constexpr int COV_MAX_DIM = 1024;

}  // namespace dss

using namespace dss;

extern "C" int dss_segment_bboxes(const uint8_t* segmaps, int B, int H, int W, int num_erode, int num_dilate, int* boxes,
                                  uint8_t* present, dss_stream_t stream) {
  DSS_REQUIRE(segmaps && boxes && present, "segment_bboxes: null pointer");
  DSS_REQUIRE(B > 0 && H > 0 && W > 0, "segment_bboxes: empty problem B=%d H=%d W=%d", B, H, W);
  DSS_REQUIRE(num_erode >= 0 && num_dilate >= 0, "segment_bboxes: negative erode / dilate count");
  if ((long long)H * W > BB_MAX_PIXELS) {
    set_error("segment_bboxes: %d x %d grid exceeds %d cells", H, W, BB_MAX_PIXELS);
    return DSS_ERR_UNSUPPORTED;
  }
  DSS_REQUIRE((long long)B * 256 < (1ll << 31), "segment_bboxes: too many images in one call (%d)", B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LaunchScope scope(st, KC_MISC);
  segment_bbox_kernel<<<B * 256, BB_THREADS, 2 * H * W, st>>>(segmaps, H, W, num_erode, num_dilate, boxes, present);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

extern "C" size_t dss_covariance_workspace_bytes(int M, int d) {
  if (M < 2 || d < 1 || d > COV_MAX_DIM) return 0;
  return cov_layout(M, d).total;
}

extern "C" int dss_covariance(const float* X, int M, int d, float* mean, float* cov, int ldc, void* ws, size_t ws_bytes,
                              dss_stream_t stream) {
  DSS_REQUIRE(X && mean && cov && ws, "covariance: null pointer");
  DSS_REQUIRE(M >= 2 && d >= 1, "covariance: need at least 2 rows and 1 column (M=%d d=%d)", M, d);
  DSS_REQUIRE(ldc >= d, "covariance: ldc (%d) < d (%d)", ldc, d);
  DSS_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "covariance: workspace must be 256-byte aligned");
  if (d > COV_MAX_DIM) {
    set_error("covariance: d=%d exceeds %d", d, COV_MAX_DIM);
    return DSS_ERR_UNSUPPORTED;
  }
  const CovLayout L = cov_layout(M, d);
  if (ws_bytes < L.total) {
    set_error("covariance: workspace too small (%zu < %zu)", ws_bytes, L.total);
    return DSS_ERR_WORKSPACE;
  }
  uint8_t* w = static_cast<uint8_t*>(ws);
  double* colpart = reinterpret_cast<double*>(w);
  unsigned* maxabs = reinterpret_cast<unsigned*>(w + L.off_maxabs);
  double* mean64 = reinterpret_cast<double*>(w + L.off_mean);
  double* part = reinterpret_cast<double*>(w + L.off_part);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  { LaunchScope scope(st, KC_MISC); colstats_kernel<<<L.Gc, CL_THREADS, 0, st>>>(X, M, d, L.rows_c, colpart, maxabs); }
  { LaunchScope scope(st, KC_MISC); column_mean_kernel<<<1, CL_THREADS, 0, st>>>(colpart, L.Gc, M, d, mean64, mean); }
  {
    LaunchScope scope(st, KC_MISC);
    covariance_tile_kernel<<<dim3(L.nt, L.splits), CL_THREADS, 0, st>>>(X, M, d, mean64, L.rows_split, part);
  }
  { LaunchScope scope(st, KC_MISC); covariance_combine_kernel<<<L.nt, CL_THREADS, 0, st>>>(part, L.splits, M, d, cov, ldc); }
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

extern "C" int dss_pca_project(const float* X, int M, int d, const float* mean, const float* V, int p, float* Y,
                               dss_stream_t stream) {
  DSS_REQUIRE(X && mean && V && Y, "pca_project: null pointer");
  DSS_REQUIRE(M >= 1 && d >= 1 && p >= 1, "pca_project: empty problem (M=%d d=%d p=%d)", M, d, p);
  if (p > 64) {
    set_error("pca_project: p=%d exceeds 64", p);
    return DSS_ERR_UNSUPPORTED;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LaunchScope scope(st, KC_MISC);
  pca_project_kernel<<<cdiv(M, 64), CL_THREADS, 0, st>>>(X, M, d, mean, V, p, Y);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

extern "C" size_t dss_kmeans_workspace_bytes(int M, int dims, int k) {
  if (M < 1 || dims < 1 || k < 1 || !km_supported(dims, k)) return 0;
  return km_layout(M, dims, k).total;
}

extern "C" int dss_kmeans(const float* X, int M, int dims, int k, unsigned int seed, int max_iter, float tol,
                          float* centers, int* labels, int* info, float* inertia, void* ws, size_t ws_bytes,
                          dss_stream_t stream) {
  DSS_REQUIRE(X && centers && labels && info && ws, "kmeans: null pointer");
  DSS_REQUIRE(M >= 1 && dims >= 1 && k >= 1, "kmeans: empty problem (M=%d dims=%d k=%d)", M, dims, k);
  DSS_REQUIRE(k <= M, "kmeans: k=%d > %d points", k, M);
  DSS_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "kmeans: workspace must be 256-byte aligned");
  if (!km_supported(dims, k)) {
    set_error("kmeans: k=%d at dims=%d is not supported (k <= 64 at dims <= 768, or k <= 256 at dims <= 64)", k, dims);
    return DSS_ERR_UNSUPPORTED;
  }
  const KmLayout L = km_layout(M, dims, k);
  if (ws_bytes < L.total) {
    set_error("kmeans: workspace too small (%zu < %zu)", ws_bytes, L.total);
    return DSS_ERR_WORKSPACE;
  }
  uint8_t* w = static_cast<uint8_t*>(ws);
  KmParams p;
  p.X = X; p.M = M; p.dims = dims; p.k = k; p.trials = kmeans_local_trials(k);
  p.max_iter = max_iter > 0 ? max_iter : 300;
  p.tol = tol >= 0.f ? tol : 1e-4f;
  p.seed = seed;
  p.st = reinterpret_cast<KmState*>(w);
  p.colpart = reinterpret_cast<double*>(w + L.off_colpart);
  p.maxabs = reinterpret_cast<unsigned*>(w + L.off_maxabs);
  p.Gc = L.Gc; p.rows_c = L.rows_c;
  p.mind2 = reinterpret_cast<float*>(w + L.off_mind2);
  p.chunksum = reinterpret_cast<double*>(w + L.off_chunk);
  p.potpart = reinterpret_cast<double*>(w + L.off_pot);
  p.inpart = reinterpret_cast<double*>(w + L.off_inpart);
  p.G = L.G;
  p.accs = reinterpret_cast<long long*>(w + L.off_accs);
  p.cnts = reinterpret_cast<int*>(w + L.off_cnts);
  p.tot = reinterpret_cast<long long*>(w + L.off_tot);
  p.cnt = reinterpret_cast<int*>(w + L.off_cnt);
  p.Gp = L.Gp; p.rows_p = L.rows_p; p.DT = L.DT;
  p.centers = centers; p.labels = labels;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DSS_CHECK_CUDA(cudaMemsetAsync(p.st, 0, sizeof(KmState), st));
  DSS_CHECK_CUDA(cudaMemsetAsync(p.maxabs, 0, 4, st));
  DSS_CHECK_CUDA(cudaMemsetAsync(labels, 0xFF, (size_t)M * 4, st));   // -1: the first E step changes every label
  const size_t cen_smem = (size_t)k * dims * 4;
  const size_t acc_smem = (size_t)k * L.DT * 8 + (size_t)k * 4;
  const int nDT = cdiv(dims, L.DT);
  const int nj = cdiv(dims, 32);
  if (nj <= 1) return km_run<1>(p, cen_smem, acc_smem, nDT, st, info, inertia);
  if (nj <= 2) return km_run<2>(p, cen_smem, acc_smem, nDT, st, info, inertia);
  if (nj <= 4) return km_run<4>(p, cen_smem, acc_smem, nDT, st, info, inertia);
  if (nj <= 8) return km_run<8>(p, cen_smem, acc_smem, nDT, st, info, inertia);
  if (nj <= 12) return km_run<12>(p, cen_smem, acc_smem, nDT, st, info, inertia);
  return km_run<24>(p, cen_smem, acc_smem, nDT, st, info, inertia);
}
