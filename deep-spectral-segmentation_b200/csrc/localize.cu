// Object localization boxes (replace get_bbox_from_patch_mask + get_largest_cc_box, lost + patch_scoring + detect_box
// and dino_seg of the reference's object-localization/object_discovery.py).
//
// All three run one CTA per image on a patch grid of at most LOC_MAX_CELLS cells held in shared memory, and share one
// connected-components routine: lock-free union-find whose links go from the larger root to the smaller one with
// atomicMin, then path compression. Every component's root is therefore its smallest raster index, which is the order
// in which scipy.ndimage.label and skimage.measure.label number components (by the raster position of their first
// pixel): "label l" of the reference is "the l-th smallest root" here. Sizes and extents come from shared-memory
// integer atomics, so the result does not depend on thread scheduling.
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace dss {

constexpr int LOC_THREADS = 1024;
constexpr int LOC_MAX_CELLS = 128 * 128;

static inline int next_pow2(int n) {
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

__device__ __forceinline__ int cc_find(const volatile int* parent, int x) {
  int p;
  while ((p = parent[x]) != x) x = p;
  return x;
}

// Joins the components of a and b: the larger root is linked under the smaller one. A failed atomicMin means the
// larger root was linked meanwhile; its new parent is then joined with b.
__device__ __forceinline__ void cc_union(int* parent, int a, int b) {
  while (true) {
    a = cc_find(parent, a);
    b = cc_find(parent, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(&parent[a], b);
    if (old == a) return;
    a = old;
  }
}

// parent[i] = root (smallest raster index) of cell i's component, -1 for cells with mask[i] == 0;
// size[r] = cell count of the component rooted at r (undefined for non-roots). conn8: 8-connectivity, else 4.
__device__ void cc_label(const uint8_t* mask, int* parent, int* size, int gh, int gw, bool conn8) {
  const int n = gh * gw;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    parent[i] = mask[i] ? i : -1;
    size[i] = 0;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    if (!mask[i]) continue;
    const int r = i / gw, c = i - r * gw;
    if (c > 0 && mask[i - 1]) cc_union(parent, i, i - 1);
    if (r > 0) {
      if (mask[i - gw]) cc_union(parent, i, i - gw);
      if (conn8 && c > 0 && mask[i - gw - 1]) cc_union(parent, i, i - gw - 1);
      if (conn8 && c < gw - 1 && mask[i - gw + 1]) cc_union(parent, i, i - gw + 1);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (mask[i]) parent[i] = cc_find(parent, i);
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (mask[i]) atomicAdd(&size[parent[i]], 1);
  __syncthreads();
}

// Ascending bitonic sort of keys[0, n2), n2 >= N a power of two chosen by the host (callers pad with ~0).
__device__ void bitonic_sort_u64(unsigned long long* keys, int n2) {
  for (int k = 2; k <= n2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n2; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], b = keys[ixj];
          if ((a > b) == ((i & k) == 0)) { keys[i] = b; keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
}

// {xmin, ymin, xmax + 1, ymax + 1} (grid units) of the cells with parent[i] == sel (sel == -1: the background cells).
// Returns false if there is no such cell.
__device__ bool cc_box(const int* parent, int gh, int gw, int sel, int* sbox) {
  const int n = gh * gw;
  if (threadIdx.x == 0) { sbox[0] = gw; sbox[1] = gh; sbox[2] = -1; sbox[3] = -1; }
  __syncthreads();
  int x0 = gw, y0 = gh, x1 = -1, y1 = -1;
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (parent[i] == sel) {
      const int r = i / gw, c = i - r * gw;
      x0 = min(x0, c); y0 = min(y0, r); x1 = max(x1, c); y1 = max(y1, r);
    }
  if (x1 >= 0) { atomicMin(&sbox[0], x0); atomicMin(&sbox[1], y0); atomicMax(&sbox[2], x1); atomicMax(&sbox[3], y1); }
  __syncthreads();
  const bool any = sbox[2] >= 0;
  __syncthreads();
  return any;
}

// The root of the largest component, ties to the smallest root (np.argmax over labels in root order); roots >= skip
// are not candidates. -1 if there is none.
__device__ int cc_largest(const int* parent, const int* size, int n, int skip, unsigned long long* sbest) {
  if (threadIdx.x == 0) *sbest = 0ull;
  __syncthreads();
  unsigned long long best = 0ull;
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (parent[i] == i && i < skip) {
      const unsigned long long key = ((unsigned long long)size[i] << 32) | (unsigned)(0x7fffffff - i);
      best = key > best ? key : best;
    }
  if (best) atomicMax(sbest, best);
  __syncthreads();
  const unsigned long long b = *sbest;
  __syncthreads();
  return b ? 0x7fffffff - (int)(b & 0xffffffffu) : -1;
}

struct EigsegImage { int P, gh, gw, H, W, ok; };

// One image of LOST or DINO-seg: N = gh gw cells, n2 = next_pow2(N) sort keys, un-padded size H x W (LOST). A uniform
// batch passes one descriptor by value (imgs == NULL); a ragged batch a table of B. Image b's rows start at row
// b * pitch of the inputs (pitch = N, or n_max of a padded ragged batch).
struct LocImage { int N, n2, gh, gw, H, W; };
__device__ __forceinline__ LocImage loc_image(const LocImage* imgs, const LocImage& uni, int b) {
  return imgs ? imgs[b] : uni;
}

// Shared memory of the box kernels: parent + size (or the sort keys, which they replace), the mask, LOST's list
__device__ __forceinline__ void loc_carve(int n, int n2, unsigned char* smem, unsigned long long** keys, int** parent,
                                          int** size, uint8_t** mask, int** list) {
  const size_t rbytes = (size_t)(n2 > n ? n2 : n) * 8;
  *keys = reinterpret_cast<unsigned long long*>(smem);
  *parent = reinterpret_cast<int*>(smem);
  *size = reinterpret_cast<int*>(smem) + n;
  *mask = smem + rbytes;
  *list = reinterpret_cast<int*>(smem + rbytes + ((size_t)n + 15) / 16 * 16);
}

static size_t loc_smem_bytes(int n, int n2, bool with_list) {
  const size_t rbytes = (size_t)(n2 > n ? n2 : n) * 8;
  return rbytes + ((size_t)n + 15) / 16 * 16 + (with_list ? (size_t)n * 4 : 0);
}

// ---- a) eigen-segmentation boxes (get_bbox_from_patch_mask, object_discovery.py:85-126)
__global__ void __launch_bounds__(LOC_THREADS)
eigseg_box_kernel(const float* __restrict__ evecs, int K, int N, int which, const EigsegImage* __restrict__ imgs,
                  int* __restrict__ boxes, int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int sbox[4];
  __shared__ int scount;
  __shared__ unsigned long long sbest;
  const int b = blockIdx.x;
  const EigsegImage im = imgs[b];
  if (!im.ok) {
    if (threadIdx.x == 0) {
      status[b] = DSS_LOC_NO_GRID;
      for (int j = 0; j < 4; ++j) boxes[b * 4 + j] = 0;
    }
    return;
  }
  unsigned long long* keys; int *parent, *size, *list; uint8_t* mask;
  loc_carve(N, N, smem, &keys, &parent, &size, &mask, &list);
  const float* v = evecs + ((long long)b * K + which) * N;
  if (threadIdx.x == 0) scount = 0;
  __syncthreads();
  int cnt = 0;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const uint8_t m = v[i] > 0.f;
    mask[i] = m;
    cnt += m;
  }
  atomicAdd(&scount, cnt);
  __syncthreads();
  // 0.5 < mean < 1 (exact in float64 for these N) or an empty mask: the complement is the object
  const int s = scount;
  if ((2 * s > N && s < N) || s == 0)
    for (int i = threadIdx.x; i < N; i += blockDim.x) mask[i] = 1 - mask[i];
  __syncthreads();
  cc_label(mask, parent, size, im.gh, im.gw, true);   // skimage.measure.label: connectivity = ndim (8-connected)
  const int root = cc_largest(parent, size, N, N, &sbest);   // never -1: the mask is not empty after the flip
  cc_box(parent, im.gh, im.gw, root, sbox);
  if (threadIdx.x == 0) {
    const int P = im.P;
    boxes[b * 4 + 0] = sbox[0] * P;
    boxes[b * 4 + 1] = sbox[1] * P;
    boxes[b * 4 + 2] = min((sbox[2] + 1) * P, im.W);
    boxes[b * 4 + 3] = min((sbox[3] + 1) * P, im.H);
    status[b] = DSS_LOC_OK;
  }
}

// ---- b) LOST (lost + patch_scoring + detect_box, object_discovery.py:129-227)
// degree[b, i] = #{j != i : A[b, i, j] > 0} over image b's N cells: one warp per row
__global__ void __launch_bounds__(256)
lost_degree_kernel(const float* __restrict__ A, const LocImage* __restrict__ imgs, LocImage uni, int pitch, int ldw,
                   int* __restrict__ degree) {
  const int b = blockIdx.y, row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int N = loc_image(imgs, uni, b).N;
  if (row >= N) return;
  const float* a = A + ((long long)b * pitch + row) * ldw;
  int c = 0;
  for (int j = lane; j < N; j += 32) c += (j != row) && (a[j] > 0.f);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) degree[(long long)b * pitch + row] = c;
}

__global__ void __launch_bounds__(LOC_THREADS)
lost_box_kernel(const float* __restrict__ A, const LocImage* __restrict__ imgs, LocImage uni, int pitch, int ldw,
                const int* __restrict__ degree, int P, int k_patches, int* __restrict__ boxes, int* __restrict__ seeds,
                int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int sbox[4];
  __shared__ int snsim;
  const int b = blockIdx.x;
  const LocImage im = loc_image(imgs, uni, b);
  const int N = im.N, n2 = im.n2, gh = im.gh, gw = im.gw, H = im.H, W = im.W;
  unsigned long long* keys; int *parent, *size, *list; uint8_t* mask;
  loc_carve(N, n2, smem, &keys, &parent, &size, &mask, &list);
  const float* Ab = A + (long long)b * pitch * ldw;
  // ascending degree, ties by patch index (a stable order; torch.argsort(stable=False) leaves ties unspecified)
  for (int i = threadIdx.x; i < n2; i += blockDim.x)
    keys[i] = i < N ? ((unsigned long long)degree[(long long)b * pitch + i] << 32) | (unsigned)i : ~0ull;
  __syncthreads();
  bitonic_sort_u64(keys, n2);
  const int seed = (int)(keys[0] & 0xffffffffu);
  const int kk = min(k_patches, N);
  // similars: potentials (the first kk in that order) with A[seed, p] > 0, compacted in order by warp 0
  if (threadIdx.x < 32) {
    int base = 0;
    for (int t0 = 0; t0 < kk; t0 += 32) {
      const int t = t0 + threadIdx.x;
      int p = 0;
      bool keep = false;
      if (t < kk) {
        p = (int)(keys[t] & 0xffffffffu);
        keep = Ab[(long long)seed * ldw + p] > 0.f;
      }
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
      if (keep) list[base + __popc(bal & ((1u << threadIdx.x) - 1u))] = p;
      base += __popc(bal);
    }
    if (threadIdx.x == 0) snsim = base;
  }
  __syncthreads();
  // M[j] = sum over the similars, in order, of A[s, j] (fp32); the sort keys are dead from here on
  const int nsim = snsim;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    float m = 0.f;
    for (int t = 0; t < nsim; ++t) m += Ab[(long long)list[t] * ldw + j];
    mask[j] = m > 0.f;
  }
  __syncthreads();
  cc_label(mask, parent, size, gh, gw, false);   // scipy.ndimage.label's default cross: 4-connected
  const int cc = parent[seed];
  if (cc < 0) {
    if (threadIdx.x == 0) {
      status[b] = DSS_LOC_SEED_IN_BACKGROUND;
      for (int j = 0; j < 4; ++j) boxes[b * 4 + j] = 0;
      if (seeds) seeds[b] = seed;
    }
    return;
  }
  cc_box(parent, gh, gw, cc, sbox);
  if (threadIdx.x == 0) {
    boxes[b * 4 + 0] = sbox[0] * P;
    boxes[b * 4 + 1] = sbox[1] * P;
    boxes[b * 4 + 2] = min((sbox[2] + 1) * P, W);
    boxes[b * 4 + 3] = min((sbox[3] + 1) * P, H);
    status[b] = DSS_LOC_OK;
    if (seeds) seeds[b] = seed;
  }
}

// ---- c) DINO-seg (dino_seg, object_discovery.py:230-277)
__device__ __forceinline__ unsigned f32_order_key(float x) {
  const unsigned u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(LOC_THREADS)
dinoseg_box_kernel(const float* __restrict__ attn, int heads, const LocImage* __restrict__ imgs, LocImage uni, int pitch,
                   int head, int P, int* __restrict__ boxes, int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int sbox[4];
  __shared__ int smaxroot, scomp;
  __shared__ float ssum;
  __shared__ unsigned long long sbest;
  __shared__ double red[LOC_THREADS / 32];
  const int b = blockIdx.x;
  const LocImage im = loc_image(imgs, uni, b);
  const int N = im.N, n2 = im.n2, gh = im.gh, gw = im.gw;
  unsigned long long* keys; int *parent, *size, *list; uint8_t* mask;
  loc_carve(N, n2, smem, &keys, &parent, &size, &mask, &list);
  const float* a = attn + ((long long)b * heads + head) * pitch;
  // torch.sort ascending (ties by index), val /= sum(val), cumsum, keep where the cumulative mass > 1 - 0.6
  double part = 0.0;
  for (int i = threadIdx.x; i < n2; i += blockDim.x) {
    if (i < N) {
      const float x = a[i];
      keys[i] = ((unsigned long long)f32_order_key(x) << 32) | (unsigned)i;
      part += (double)x;
    } else {
      keys[i] = ~0ull;
    }
  }
  part = warp_sum(part);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    ssum = (float)s;
  }
  bitonic_sort_u64(keys, n2);
  if (threadIdx.x == 0) {
    // torch's CPU cumsum: one pass in order, a double accumulator, every prefix rounded to float
    const float sum = ssum, thr = (float)(1.0 - 0.6);
    double acc = 0.0;
    for (int p = 0; p < N; ++p) {
      const int idx = (int)(keys[p] & 0xffffffffu);
      acc += (double)(a[idx] / sum);
      mask[idx] = (float)acc > thr;
    }
  }
  __syncthreads();
  cc_label(mask, parent, size, gh, gw, false);
  // the reference sizes labels 0 .. n-1 only (range(max(label))): with n >= 2 components the largest of labels
  // 1 .. n-1 wins (the last-numbered component n never does); with n <= 1 it takes label 0, the background cells
  if (threadIdx.x == 0) { smaxroot = -1; scomp = 0; }
  __syncthreads();
  int mr = -1, nroots = 0;
  for (int i = threadIdx.x; i < N; i += blockDim.x)
    if (parent[i] == i) { mr = max(mr, i); ++nroots; }
  if (nroots) { atomicMax(&smaxroot, mr); atomicAdd(&scomp, nroots); }
  __syncthreads();
  const int sel = scomp >= 2 ? cc_largest(parent, size, N, smaxroot, &sbest) : -1;
  const bool any = cc_box(parent, gh, gw, sel, sbox);
  if (threadIdx.x == 0) {
    if (!any) {
      status[b] = DSS_LOC_EMPTY_COMPONENT;
      for (int j = 0; j < 4; ++j) boxes[b * 4 + j] = 0;
    } else {
      boxes[b * 4 + 0] = sbox[0] * P;
      boxes[b * 4 + 1] = sbox[1] * P;
      boxes[b * 4 + 2] = (sbox[2] + 1) * P;
      boxes[b * 4 + 3] = (sbox[3] + 1) * P;
      status[b] = DSS_LOC_OK;
    }
  }
}

static int loc_set_smem(const void* fn, size_t smem) {
  DSS_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return DSS_OK;
}

// The reference's four patch-grid cases, tried in order (object_discovery.py:88-99)
static EigsegImage eigseg_grid(int N, int H, int W) {
  EigsegImage e{0, 0, 0, H, W, 1};
  if ((H / 8) * (W / 8) == N) { e.P = 8; e.gh = H / 8; e.gw = W / 8; }
  else if ((H / 16) * (W / 16) == N) { e.P = 16; e.gh = H / 16; e.gw = W / 16; }
  else if (4 * (H / 16) * (W / 16) == N) { e.P = 8; e.gh = 2 * (H / 16); e.gw = 2 * (W / 16); }
  else if (16 * (H / 32) * (W / 32) == N) { e.P = 8; e.gh = 4 * (H / 32); e.gw = 4 * (W / 32); }
  else e.ok = 0;
  return e;
}

static LocImage loc_image_host(int gh, int gw, int H, int W) {
  const int N = gh * gw;
  return {N, next_pow2(N), gh, gw, H, W};
}

// LOST over B images (imgs: device table, or NULL and every image `uni`); shared memory for max_n cells
static int launch_lost(const float* A, int B, int pitch, int ldw, const LocImage* imgs, const LocImage& uni, int max_n,
                       int P, int k_patches, int* boxes, int* seeds, int* status, int* degree, cudaStream_t st) {
  {
    LaunchScope scope(st, KC_MISC);
    lost_degree_kernel<<<dim3(cdiv(max_n, 8), B), 256, 0, st>>>(A, imgs, uni, pitch, ldw, degree);
    DSS_CHECK_CUDA(cudaGetLastError());
  }
  const size_t smem = loc_smem_bytes(max_n, next_pow2(max_n), true);
  int rc;
  if ((rc = loc_set_smem((const void*)lost_box_kernel, smem))) return rc;
  LaunchScope scope(st, KC_MISC);
  lost_box_kernel<<<B, LOC_THREADS, smem, st>>>(A, imgs, uni, pitch, ldw, degree, P, k_patches, boxes, seeds, status);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

static int launch_dinoseg(const float* attn, int B, int heads, int pitch, int head, const LocImage* imgs,
                          const LocImage& uni, int max_n, int P, int* boxes, int* status, cudaStream_t st) {
  const size_t smem = loc_smem_bytes(max_n, next_pow2(max_n), false);
  int rc;
  if ((rc = loc_set_smem((const void*)dinoseg_box_kernel, smem))) return rc;
  LaunchScope scope(st, KC_MISC);
  dinoseg_box_kernel<<<B, LOC_THREADS, smem, st>>>(attn, heads, imgs, uni, pitch, head, P, boxes, status);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

// The descriptors of a ragged batch from dims_host [B, per] = {gh, gw[, H, W]}: every grid non-empty, at most n_max
// and LOC_MAX_CELLS cells. Returns the largest N_b in *max_n.
static int ragged_loc_images(const char* name, const int* dims, int B, int per, int n_max, std::vector<LocImage>& imgs,
                             int* max_n) {
  imgs.resize(B);
  *max_n = 0;
  for (int b = 0; b < B; ++b) {
    const int* d = dims + (size_t)b * per;
    const int gh = d[0], gw = d[1], H = per == 4 ? d[2] : 1, W = per == 4 ? d[3] : 1;
    DSS_REQUIRE(gh > 0 && gw > 0 && H > 0 && W > 0, "%s: image %d has grid %dx%d, size %dx%d", name, b, gh, gw, H, W);
    const long long N = (long long)gh * gw;
    DSS_REQUIRE(N <= n_max, "%s: image %d's %dx%d grid has more than n_max = %d cells", name, b, gh, gw, n_max);
    if (N > LOC_MAX_CELLS) {
      set_error("%s: image %d's %lld cells exceed the %d (128 x 128) a CTA holds in shared memory", name, b, N,
                LOC_MAX_CELLS);
      return DSS_ERR_UNSUPPORTED;
    }
    imgs[b] = loc_image_host(gh, gw, H, W);
    *max_n = std::max(*max_n, (int)N);
  }
  return DSS_OK;
}

}  // namespace dss

using namespace dss;

extern "C" size_t dss_eigseg_boxes_workspace_bytes(int B) {
  return B > 0 ? align_up((size_t)B * sizeof(EigsegImage), 256) : 0;
}

extern "C" int dss_eigseg_boxes(const float* evecs, int B, int K, int N, int which, const int* dims_host, int* boxes,
                                int* status, void* ws, size_t ws_bytes, dss_stream_t stream) {
  DSS_REQUIRE(evecs && dims_host && boxes && status && ws, "eigseg_boxes: null pointer");
  DSS_REQUIRE(B > 0 && N > 0 && which >= 0 && which < K, "eigseg_boxes: bad shape / row (B=%d K=%d N=%d which=%d)", B,
              K, N, which);
  if (N > LOC_MAX_CELLS) {
    set_error("eigseg_boxes: %d cells exceed the %d (128 x 128) a CTA holds in shared memory", N, LOC_MAX_CELLS);
    return DSS_ERR_UNSUPPORTED;
  }
  if (ws_bytes < dss_eigseg_boxes_workspace_bytes(B)) {
    set_error("eigseg_boxes: workspace too small (%zu < %zu)", ws_bytes, dss_eigseg_boxes_workspace_bytes(B));
    return DSS_ERR_WORKSPACE;
  }
  std::vector<EigsegImage> imgs(B);
  for (int b = 0; b < B; ++b) {
    DSS_REQUIRE(dims_host[2 * b] > 0 && dims_host[2 * b + 1] > 0, "eigseg_boxes: image %d has size %dx%d", b,
                dims_host[2 * b], dims_host[2 * b + 1]);
    imgs[b] = eigseg_grid(N, dims_host[2 * b], dims_host[2 * b + 1]);
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // pageable source: the copy is staged before cudaMemcpyAsync returns, so `imgs` may go out of scope
  DSS_CHECK_CUDA(cudaMemcpyAsync(ws, imgs.data(), (size_t)B * sizeof(EigsegImage), cudaMemcpyHostToDevice, st));
  const size_t smem = loc_smem_bytes(N, N, false);
  int rc;
  if ((rc = loc_set_smem((const void*)eigseg_box_kernel, smem))) return rc;
  LaunchScope scope(st, KC_MISC);
  eigseg_box_kernel<<<B, LOC_THREADS, smem, st>>>(evecs, K, N, which, reinterpret_cast<const EigsegImage*>(ws), boxes,
                                                  status);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

extern "C" size_t dss_lost_workspace_bytes(int B, int N) {
  return (B > 0 && N > 0) ? align_up((size_t)B * N * sizeof(int), 256) : 0;
}

extern "C" int dss_lost_boxes(const float* A, int B, int N, int ldw, int grid_h, int grid_w, int H, int W, int P,
                              int k_patches, int* boxes, int* seeds, int* status, void* ws, size_t ws_bytes,
                              dss_stream_t stream) {
  DSS_REQUIRE(A && boxes && status && ws, "lost_boxes: null pointer");
  DSS_REQUIRE(B > 0 && N > 0 && ldw >= N && grid_h > 0 && grid_w > 0 && grid_h * grid_w == N,
              "lost_boxes: bad shape (B=%d N=%d ldw=%d grid %dx%d)", B, N, ldw, grid_h, grid_w);
  DSS_REQUIRE(P > 0 && H > 0 && W > 0 && k_patches > 0, "lost_boxes: bad image size / patch / k_patches");
  if (N > LOC_MAX_CELLS) {
    set_error("lost_boxes: %d cells exceed the %d (128 x 128) a CTA holds in shared memory", N, LOC_MAX_CELLS);
    return DSS_ERR_UNSUPPORTED;
  }
  if (ws_bytes < dss_lost_workspace_bytes(B, N)) {
    set_error("lost_boxes: workspace too small (%zu < %zu)", ws_bytes, dss_lost_workspace_bytes(B, N));
    return DSS_ERR_WORKSPACE;
  }
  return launch_lost(A, B, N, ldw, nullptr, loc_image_host(grid_h, grid_w, H, W), N, P, k_patches, boxes, seeds, status,
                     reinterpret_cast<int*>(ws), static_cast<cudaStream_t>(stream));
}

extern "C" size_t dss_lost_ragged_workspace_bytes(int B, int n_max) {
  return (B > 0 && n_max > 0) ? align_up((size_t)B * n_max * sizeof(int), 256) + align_up(B * sizeof(LocImage), 256)
                              : 0;
}

extern "C" int dss_lost_boxes_ragged(const float* A, int B, int n_max, int ldw, const int* dims_host, int P,
                                     int k_patches, int* boxes, int* seeds, int* status, void* ws, size_t ws_bytes,
                                     dss_stream_t stream) {
  DSS_REQUIRE(A && dims_host && boxes && status && ws, "lost_boxes_ragged: null pointer");
  DSS_REQUIRE(B > 0 && n_max > 0 && ldw >= n_max, "lost_boxes_ragged: bad shape (B=%d n_max=%d ldw=%d)", B, n_max, ldw);
  DSS_REQUIRE(P > 0 && k_patches > 0, "lost_boxes_ragged: bad patch / k_patches");
  std::vector<LocImage> imgs;
  int max_n, rc;
  if ((rc = ragged_loc_images("lost_boxes_ragged", dims_host, B, 4, n_max, imgs, &max_n))) return rc;
  const size_t need = dss_lost_ragged_workspace_bytes(B, n_max), deg_bytes = align_up((size_t)B * n_max * 4, 256);
  if (ws_bytes < need) {
    set_error("lost_boxes_ragged: workspace too small (%zu < %zu)", ws_bytes, need);
    return DSS_ERR_WORKSPACE;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* tab = reinterpret_cast<uint8_t*>(ws) + deg_bytes;
  // pageable source: the copy is staged before cudaMemcpyAsync returns, so `imgs` may go out of scope
  DSS_CHECK_CUDA(cudaMemcpyAsync(tab, imgs.data(), (size_t)B * sizeof(LocImage), cudaMemcpyHostToDevice, st));
  return launch_lost(A, B, n_max, ldw, reinterpret_cast<const LocImage*>(tab), imgs[0], max_n, P, k_patches, boxes,
                     seeds, status, reinterpret_cast<int*>(ws), st);
}

extern "C" int dss_dinoseg_boxes(const float* cls_attn, int B, int heads, int N, int head, int grid_h, int grid_w, int P,
                                 int* boxes, int* status, dss_stream_t stream) {
  DSS_REQUIRE(cls_attn && boxes && status, "dinoseg_boxes: null pointer");
  DSS_REQUIRE(B > 0 && heads > 0 && N > 0 && grid_h > 0 && grid_w > 0 && grid_h * grid_w == N,
              "dinoseg_boxes: bad shape (B=%d heads=%d N=%d grid %dx%d)", B, heads, N, grid_h, grid_w);
  DSS_REQUIRE(head >= 0 && head < heads, "dinoseg_boxes: head %d not in [0, %d)", head, heads);
  DSS_REQUIRE(P > 0, "dinoseg_boxes: bad patch size %d", P);
  if (N > LOC_MAX_CELLS) {
    set_error("dinoseg_boxes: %d cells exceed the %d (128 x 128) a CTA holds in shared memory", N, LOC_MAX_CELLS);
    return DSS_ERR_UNSUPPORTED;
  }
  return launch_dinoseg(cls_attn, B, heads, N, head, nullptr, loc_image_host(grid_h, grid_w, 1, 1), N, P, boxes, status,
                        static_cast<cudaStream_t>(stream));
}

extern "C" size_t dss_dinoseg_ragged_workspace_bytes(int B) {
  return B > 0 ? align_up((size_t)B * sizeof(LocImage), 256) : 0;
}

extern "C" int dss_dinoseg_boxes_ragged(const float* cls_attn, int B, int heads, int n_max, int head,
                                        const int* dims_host, int P, int* boxes, int* status, void* ws, size_t ws_bytes,
                                        dss_stream_t stream) {
  DSS_REQUIRE(cls_attn && dims_host && boxes && status && ws, "dinoseg_boxes_ragged: null pointer");
  DSS_REQUIRE(B > 0 && heads > 0 && n_max > 0, "dinoseg_boxes_ragged: bad shape (B=%d heads=%d n_max=%d)", B, heads,
              n_max);
  DSS_REQUIRE(head >= 0 && head < heads, "dinoseg_boxes_ragged: head %d not in [0, %d)", head, heads);
  DSS_REQUIRE(P > 0, "dinoseg_boxes_ragged: bad patch size %d", P);
  std::vector<LocImage> imgs;
  int max_n, rc;
  if ((rc = ragged_loc_images("dinoseg_boxes_ragged", dims_host, B, 2, n_max, imgs, &max_n))) return rc;
  if (ws_bytes < dss_dinoseg_ragged_workspace_bytes(B)) {
    set_error("dinoseg_boxes_ragged: workspace too small (%zu < %zu)", ws_bytes, dss_dinoseg_ragged_workspace_bytes(B));
    return DSS_ERR_WORKSPACE;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DSS_CHECK_CUDA(cudaMemcpyAsync(ws, imgs.data(), (size_t)B * sizeof(LocImage), cudaMemcpyHostToDevice, st));
  return launch_dinoseg(cls_attn, B, heads, n_max, head, reinterpret_cast<const LocImage*>(ws), imgs[0], max_n, P, boxes,
                        status, st);
}
