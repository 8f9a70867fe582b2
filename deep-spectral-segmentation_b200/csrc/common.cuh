// Shared device/host helpers for libdss_b200 (sm_90a only).
// PTX wrappers for mbarrier, TMA (cp.async.bulk.tensor), wgmma, thread-block clusters.
#pragma once
#include <cuda.h>  // CUtensorMap (types only; the driver entry point is resolved at run time, no -lcuda)
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dss_b200.h"

#if defined(__CUDA_ARCH__) && !defined(__CUDA_ARCH_FEAT_SM90_ALL)
#error "libdss_b200 is written for sm_90a only: compile with -gencode arch=compute_90a,code=sm_90a"
#endif

namespace dss {

// ---------------------------------------------------------------- host side error plumbing
void set_error(const char* fmt, ...);
const char* last_error();

#define DSS_CHECK_CUDA(expr)                                                                      \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      ::dss::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));     \
      return DSS_ERR_CUDA;                                                                        \
    }                                                                                             \
  } while (0)

#define DSS_REQUIRE(cond, ...)                                                                    \
  do {                                                                                            \
    if (!(cond)) {                                                                                \
      ::dss::set_error(__VA_ARGS__);                                                              \
      return DSS_ERR_BAD_ARG;                                                                     \
    }                                                                                             \
  } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

int device_sm_count();

// ---------------------------------------------------------------- host functions shared between files
// TMA tensor maps (gemm.cu): 128 B swizzle, 128-byte-wide boxes
int make_tmap_f16(CUtensorMap* tm, const void* ptr, int rows, int cols, int box_rows);
int make_tmap_out(CUtensorMap* tm, const void* ptr, int rows, int cols, int is_f32);
int make_tmap_out3d_f32(CUtensorMap* tm, const void* ptr, int images, int rows, int ld);
int make_tmap_out3d_f16(CUtensorMap* tm, const void* ptr, int images, int rows, int cols);
// persistent wgmma GEMMs (gemm.cu)
int gemm_tile_n();
int gemm_f16_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap* tmC, const float* bias, void* out,
                int M, int N, int K, int epi, const float* aux, int rin, int rout, cudaStream_t st, int kclass, int bn);
int gemm_f16_tc_rows(const CUtensorMap& tmA, const CUtensorMap& tmB, const float* bias, void* out, int M, int N, int K,
                     int epi, const float* aux, const int* row_map, cudaStream_t st, int kclass);
int affinity_gemm_tc(const CUtensorMap& tmS, const CUtensorMap& tmS_half, int images, int Nimg, int d, float* Wout, int ldw,
                     int ncols, const unsigned int* img_max, const unsigned int* img_absmax, const uint8_t* counts,
                     float lambda, int threshold, float* deg_part, int ld_part, cudaStream_t st,
                     unsigned long long* trace = nullptr, size_t trace_bytes = 0);
// ViT kernels (vit_kernels.cu, attention.cu). split: the operand is written in the split-fp16 format of
// DSS_VIT_PRECISION_FP32 (A order), three groups per value (split_f16 below)
int launch_im2col(const uint8_t* img, void* patches, int B, int H, int W, int P, int pad, bool split, cudaStream_t st);
int launch_layernorm(const float* x, const float* g, const float* b, void* y, int M, int d, float eps, bool split,
                     cudaStream_t st);
// qkv: f16 [B*T, 3d] (f32_keys false) or the fp32 qkv GEMM output of DSS_VIT_PRECISION_FP32 (f32_keys true)
int launch_cls_attention(const void* qkv, bool f32_keys, int B, int T, int heads, float* out, cudaStream_t st);
int launch_split_rows(const float* x, void* out, long long rows, int cols, int order, cudaStream_t st, int kclass);
int launch_gelu_split(const float* h, void* out, long long M, int n, cudaStream_t st);
int launch_qkv_split(const float* qkv, void* out, long long M, int d, cudaStream_t st);
int launch_attention_tc(const void* qkv, void* out, int B, int T, int heads, cudaStream_t st);
int launch_attention_split(const void* qkv_split, void* out, int B, int T, int heads, cudaStream_t st);

// ---- ragged ViT batches: B images of any sizes, packed one after another (vit.cu). Device table entry of image b:
// its pixels start at pixel px_off of the packed [sum H W, 3] input, its patch rows at patch_off, its T = Hp Wp + 1
// token rows (CLS first) at tok_off; stored: the stored positional grid is used unchanged (identity rule).
struct RaggedImage {
  long long px_off;
  int H, W, Hp, Wp;
  int patch_off, tok_off, stored;
};
// the image whose first row off(b) is the last one <= x (off nondecreasing in b, off(0) = 0)
template <typename Off>
__device__ __forceinline__ int ragged_find(int B, long long x, Off&& off) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((long long)off(mid) <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Where a batch's token rows lie, for the kernels outside attention that see image boundaries (attention.cu has its
// own tile locators): row0(b) is image b's first (CLS) row of the residual stream, tokens(b) its token count, and at(r)
// names positional-table row r: token t of an image with an Hp x Wp patch grid, stored = the identity rule keeps the
// stored grid.
struct PosRow { int t, Hp, Wp, stored; };
// A uniform batch: image b's T = Hp Wp + 1 rows start at b T; the positional table is the [T, d] one all images share.
struct UniformRows {
  int T, Hp, Wp, stored;
  __device__ __forceinline__ long long row0(int b) const { return (long long)b * T; }
  __device__ __forceinline__ int tokens(int) const { return T; }
  __device__ __forceinline__ PosRow at(long long r) const { return {(int)r, Hp, Wp, stored}; }
};
// A ragged batch: image b's rows start at imgs[b].tok_off; the positional table is laid out like the residual stream.
struct RaggedRows {
  const RaggedImage* imgs;
  int B;
  __device__ __forceinline__ long long row0(int b) const { return imgs[b].tok_off; }
  __device__ __forceinline__ int tokens(int b) const { return imgs[b].Hp * imgs[b].Wp + 1; }
  __device__ __forceinline__ PosRow at(long long r) const {
    const RaggedImage im = imgs[ragged_find(B, r, [&](int j) { return imgs[j].tok_off; })];
    return {(int)(r - im.tok_off), im.Hp, im.Wp, im.stored};
  }
};

// pad: the zero-padded ceil grid (imgs[b].Hp = ceil(H / P)) instead of the crop
int launch_im2col_ragged(const uint8_t* img, void* patches, const RaggedImage* imgs, int B, long long n_patches, int P,
                         bool split, bool pad, cudaStream_t st);
// The CLS attention rows of a ragged batch into out [B, heads, n_out]: image b's N_b = Hp Wp entries, then exact zeros
// up to n_out (>= every N_b)
int launch_cls_attention_ragged(const void* qkv, bool f32_keys, const RaggedImage* imgs, int B, int n_out, int heads,
                                float* out, cudaStream_t st);
// tile_prefix [B + 1]: image b's 128-query tiles are CTAs [tile_prefix[b], tile_prefix[b + 1])
int launch_attention_tc_ragged(const void* qkv, void* out, const RaggedImage* imgs, const int* tile_prefix, int B,
                               long long M, int tiles, int heads, cudaStream_t st);
int launch_attention_split_ragged(const void* qkv_split, void* out, const RaggedImage* imgs, const int* tile_prefix,
                                  int B, long long M, int tiles, int heads, cudaStream_t st);

// ---------------------------------------------------------------- launch accounting / per-class device timing
enum KernelClass {
  KC_IM2COL = 0, KC_GEMM_PATCH, KC_CLS_ROW, KC_LAYERNORM, KC_GEMM_QKV, KC_ATTENTION, KC_GEMM_PROJ, KC_GEMM_FC1,
  KC_GEMM_FC2, KC_GEMM_KPROJ, KC_GEMM_OTHER, KC_ROWNORM, KC_AFFINITY, KC_KNN, KC_EIGSH, KC_MISC, KC_COUNT
};
// Counts the launch and, when profiling is enabled, brackets it with CUDA events on the launching stream.
struct LaunchScope {
  cudaStream_t st;
  int slot;
  LaunchScope(cudaStream_t stream, int kernel_class);
  ~LaunchScope();
};

// ---------------------------------------------------------------- device helpers
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t.reg .b32 R;\n\t"
      "elect.sync R|P, 0xFFFFFFFF;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Spin on try_wait (HW-suspended probe). A bounded spin turns a protocol bug into a trap instead of a hang.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
#ifndef DSS_NO_MBAR_TIMEOUT
  uint32_t spins = 0;
#endif
  while (true) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P1;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
#ifndef DSS_NO_MBAR_TIMEOUT
    if (++spins > (1u << 24)) __trap();
#endif
  }
}

// Non-blocking probe, made warp-uniform by a vote (for event loops that watch several barriers).
__device__ __forceinline__ bool mbar_test_all(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P1;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return __all_sync(0xffffffffu, done != 0);
}

// ---- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}
// 2D tiled load global -> shared, completion signalled on an mbarrier (complete_tx::bytes).
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}

// 2D tiled store shared -> global (bulk async-group completion); rows/columns outside the tensor are clipped
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               :
               : "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
// 2D tiled reduction global += shared, performed element-wise at the L2 (residual add without reading it back)
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* tm, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.bulk_group [%0, {%2, %3}], [%1];"
               :
               : "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
// 3D tiled store (box depth 1): used for per-image matrices [B, rows, cols] so that rows are clipped per image
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tm, uint32_t smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               :
               : "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until at most N bulk groups still READ their shared-memory source (the buffers may then be reused)
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---- thread-block clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the mbarrier at this shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t rank) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}"
      ::"r"(bar), "r"(rank)
      : "memory");
}
// The same arrive without release semantics, for a consumer handing back a ring slot it has only read through wgmma
// (its reads have retired at wgmma.wait_group, so there is nothing to publish). The .release.cluster form above
// compiles to MEMBAR.ALL.GPU before every arrive, which also waits for the thread's outstanding global writes.
__device__ __forceinline__ void mbar_arrive_cluster_relaxed(uint32_t bar, uint32_t rank) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.relaxed.cluster.shared::cluster.b64 _, [ra];\n\t}"
      ::"r"(bar), "r"(rank)
      : "memory");
}
// 2D tiled load, multicast: the box lands at the same shared-memory offset in every CTA of `cta_mask`, and each
// destination CTA's mbarrier (same offset) receives the complete_tx for the bytes written into that CTA
__device__ __forceinline__ void tma_load_2d_mc(uint32_t smem_dst, const CUtensorMap* tm, uint32_t bar, int c0, int c1,
                                               uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      :
      : "r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}

// ---- wgmma (warp-group MMA): D[64 x N] (+)= A[64 x 16] * B[16 x N], fp16 operands, fp32 accumulators in registers.
// Accumulator layout (per warp w of the group, lane l): for each 8-column block i, d[4i], d[4i+1] are row 16w + l/4,
// columns 8i + 2(l%4) + {0, 1}; d[4i+2], d[4i+3] the same columns of row 16w + l/4 + 8.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Shared-memory matrix descriptor for a tile stored as rows of 128 bytes with the 128B swizzle (what a TMA box
// {64 x b16, rows} with CU_TENSOR_MAP_SWIZZLE_128B writes): 8-row groups 1024 B apart.
//   bits [0,14) start>>4 | [16,30) LBO>>4 (=1, unused for these layouts) | [32,46) SBO>>4 (=64) | [62,64) 1 = SWIZZLE_128B
// K-major operands advance K by 16 elements as +32 B of start address; an MN-major operand (B = V in P V, 64 columns
// wide) advances K by 16 rows as +2048 B.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  return (static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4)) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// Address of 16-byte chunk `chunk` (0..7) of row `row` of such a tile at `base`: the chunk index is XORed with row % 8.
__device__ __forceinline__ uint32_t sw128_addr(uint32_t base, int row, int chunk) {
  return base + row * 128 + ((chunk ^ (row & 7)) << 4);
}
// d[i .. i+7] as read-write asm operands
#define DSS_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                    "+f"(d[i + 6]), "+f"(d[i + 7])
// D[64 x 8] (+)= A(smem) * B(smem), both K-major
__device__ __forceinline__ void wgmma_m64n8_ss(float (&d)[4], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0, %1, %2, %3}, "
      "%4, %5, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 16] (+)= A(smem) * B(smem), both K-major
__device__ __forceinline__ void wgmma_m64n16_ss(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, "
      "%8, %9, p, 1, 1, 0, 0;\n\t}"
      : DSS_ACC8(0)
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 32] (+)= A(smem) * B(smem), both K-major
__device__ __forceinline__ void wgmma_m64n32_ss(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1, 0, 0;\n\t}"
      : DSS_ACC8(0), DSS_ACC8(8)
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 64] (+)= A(smem) * B(smem), both K-major
__device__ __forceinline__ void wgmma_m64n64_ss(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : DSS_ACC8(0), DSS_ACC8(8), DSS_ACC8(16), DSS_ACC8(24)
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 96] (+)= A(smem) * B(smem), both K-major
__device__ __forceinline__ void wgmma_m64n96_ss(float (&d)[48], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
      "%48, %49, p, 1, 1, 0, 0;\n\t}"
      : DSS_ACC8(0), DSS_ACC8(8), DSS_ACC8(16), DSS_ACC8(24), DSS_ACC8(32), DSS_ACC8(40)
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 128] (+)= A(smem) * B(smem), both K-major
__device__ __forceinline__ void wgmma_m64n128_ss(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : DSS_ACC8(0), DSS_ACC8(8), DSS_ACC8(16), DSS_ACC8(24), DSS_ACC8(32), DSS_ACC8(40), DSS_ACC8(48), DSS_ACC8(56)
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 192] (+)= A(smem) * B(smem), both K-major
__device__ __forceinline__ void wgmma_m64n192_ss(float (&d)[96], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, "
      "%96, %97, p, 1, 1, 0, 0;\n\t}"
      : DSS_ACC8(0), DSS_ACC8(8), DSS_ACC8(16), DSS_ACC8(24), DSS_ACC8(32), DSS_ACC8(40), DSS_ACC8(48), DSS_ACC8(56), DSS_ACC8(64), DSS_ACC8(72), DSS_ACC8(80), DSS_ACC8(88)
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 256] (+)= A(smem) * B(smem), both K-major
__device__ __forceinline__ void wgmma_m64n256_ss(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n\t}"
      : DSS_ACC8(0), DSS_ACC8(8), DSS_ACC8(16), DSS_ACC8(24), DSS_ACC8(32), DSS_ACC8(40), DSS_ACC8(48), DSS_ACC8(56), DSS_ACC8(64), DSS_ACC8(72), DSS_ACC8(80), DSS_ACC8(88), DSS_ACC8(96), DSS_ACC8(104), DSS_ACC8(112), DSS_ACC8(120)
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 64] += A(registers, the mma.sync m16n8k16 A fragment of each warp's 16 rows) * B(smem, MN-major)
__device__ __forceinline__ void wgmma_m64n64_rs_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, 1, 1, 1, 1;"
      : DSS_ACC8(0), DSS_ACC8(8), DSS_ACC8(16), DSS_ACC8(24)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc));
}
#undef DSS_ACC8
template <int N> struct Wgmma;
template <> struct Wgmma<8> { static __device__ __forceinline__ void ss(float (&d)[4], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n8_ss(d, a, b, acc); } };
template <> struct Wgmma<16> { static __device__ __forceinline__ void ss(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n16_ss(d, a, b, acc); } };
template <> struct Wgmma<32> { static __device__ __forceinline__ void ss(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n32_ss(d, a, b, acc); } };
template <> struct Wgmma<64> { static __device__ __forceinline__ void ss(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n64_ss(d, a, b, acc); } };
template <> struct Wgmma<96> { static __device__ __forceinline__ void ss(float (&d)[48], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n96_ss(d, a, b, acc); } };
template <> struct Wgmma<128> { static __device__ __forceinline__ void ss(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n128_ss(d, a, b, acc); } };
template <> struct Wgmma<192> { static __device__ __forceinline__ void ss(float (&d)[96], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n192_ss(d, a, b, acc); } };
template <> struct Wgmma<256> { static __device__ __forceinline__ void ss(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n256_ss(d, a, b, acc); } };

// per-warp-group register budget (the TMA producer group gives its registers to the MMA groups)
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t pack_h2(__half lo, __half hi) {
  __half2 h = __halves2half2(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

// one MUFU.EX2 (2 ulp), flushes denormal results to zero; exp2f would add range checks and fix-ups per element
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Split-fp16 operand format (the affinity's Gram product and the fp32-precision ViT): x = hi + lo, hi = fp16(x),
// lo = x - hi (exact in fp32, |lo| <= 2^-11 |x|), stored as the three fp16 values hi, hi/64 and 64 lo. A product of
// an A-order row [hi | hi/64 | 64 lo] with a B-order row [hi' | 64 lo' | hi'/64] is hi hi' + hi lo' + lo hi' (lo lo'
// dropped); the 2^+-6 factors keep the small terms above the fp16 subnormal range for |x| >= 2^-8 (DESIGN.md section 3).
struct SplitF16 { __half hi, hi_s, lo_s; };   // hi, hi / 64, 64 lo
__device__ __forceinline__ void split_f16(float v, __half& hi, __half& hi_s, __half& lo_s) {
  hi = __float2half_rn(v);
  const float hif = __half2float(hi);
  hi_s = __float2half_rn(hif * 0.015625f);
  lo_s = __float2half_rn((v - hif) * 64.0f);
}
__device__ __forceinline__ SplitF16 split_f16(float v) {
  SplitF16 s;
  split_f16(v, s.hi, s.hi_s, s.lo_s);
  return s;
}
// The one writer of the format: the three groups of a value (or of a pair packed by pack_h2) at o, o + stride and
// o + 2 stride, in A order [hi | hi/64 | 64 lo] (order 0) or B order [hi | 64 lo | hi/64] (order != 0).
template <typename E>
__device__ __forceinline__ void store_split(E* o, int stride, int order, E hi, E hi_s, E lo_s) {
  o[0] = hi;
  o[stride] = order ? lo_s : hi_s;
  o[2 * stride] = order ? hi_s : lo_s;
}
__device__ __forceinline__ void store_split(__half* o, int stride, int order, float v) {
  const SplitF16 s = split_f16(v);
  store_split(o, stride, order, s.hi, s.hi_s, s.lo_s);
}

// Exact-erf GELU, branch-free:  gelu(x) = x Phi(x) = relu(x) - |x| q(|x|),  q(a) = 0.5 erfc(a / sqrt 2) = 2^P(u),
// u = min(a / sqrt 2, 5), P = degree-4 minimax fit of log2(erfc(u)) - 1 on [0, 5] weighted by the error it causes in
// gelu (|x| q ln 2 dP). Max |gelu error| 6.4e-6 over the whole fp32 range, relative error <= 1e-3 for x >= -3
// (tests/test_cpu_host.py emulates this arithmetic in float32 against torch's float64 GELU); the value is then rounded
// to fp16 (relative 4.9e-4, smallest normal 6.1e-5).
// Cost per element: 7 FMA-pipe operations (bias add, scale, 4 Horner steps, final fma), one MUFU.EX2 and three ALU-pipe
// operations (sign, min, max), spread over three pipes.
#define DSS_GELU_P0 -1.0004795789718628f
#define DSS_GELU_P1 -1.6226296424865723f
#define DSS_GELU_P2 -0.9360293745994568f
#define DSS_GELU_P3 -0.12467514723539352f
#define DSS_GELU_P4 0.015465063974261284f
#define DSS_GELU_CLAMP 5.0f
__device__ __forceinline__ float gelu_erf(float x) {
  const float na = __uint_as_float(__float_as_uint(x) | 0x80000000u);   // -|x|
  const float u = fminf(__fmul_rn(na, -0.70710678118654752440f), DSS_GELU_CLAMP);
  float p = __fmaf_rn(DSS_GELU_P4, u, DSS_GELU_P3);
  p = __fmaf_rn(p, u, DSS_GELU_P2);
  p = __fmaf_rn(p, u, DSS_GELU_P1);
  p = __fmaf_rn(p, u, DSS_GELU_P0);
  return __fmaf_rn(na, ex2_approx(p), fmaxf(x, 0.f));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// LayerNorm arithmetic of one row held as float4 chunks per lane (layernorm_kernel). Every rounding is explicit (no
// contraction is left to the compiler), so the output is fixed by the source rather than by the compiler's choices:
// x - mean is one fused multiply-add on the row sum S (the mean itself is never rounded), the squares pair as
// fma(a, a, b * b), the variance is fma(Q, 1 / d, eps), and y = fma((x - mean) * rstd, gamma, beta).
__device__ __forceinline__ float ln_sum4(float4 v) { return __fadd_rn(__fadd_rn(v.x, v.y), __fadd_rn(v.z, v.w)); }
__device__ __forceinline__ float4 ln_center4(float4 v, float S, float inv_d) {
  return make_float4(__fmaf_rn(S, -inv_d, v.x), __fmaf_rn(S, -inv_d, v.y), __fmaf_rn(S, -inv_d, v.z),
                     __fmaf_rn(S, -inv_d, v.w));
}
__device__ __forceinline__ float ln_sq4(float4 a) {
  return __fadd_rn(__fmaf_rn(a.x, a.x, __fmul_rn(a.y, a.y)), __fmaf_rn(a.z, a.z, __fmul_rn(a.w, a.w)));
}
__device__ __forceinline__ float ln_rstd(float Q, float inv_d, float eps) { return rsqrtf(__fmaf_rn(Q, inv_d, eps)); }
// the four outputs of a centred chunk a
__device__ __forceinline__ float4 ln_out4(float4 a, float rstd, float4 g, float4 b) {
  return make_float4(__fmaf_rn(__fmul_rn(a.x, rstd), g.x, b.x), __fmaf_rn(__fmul_rn(a.y, rstd), g.y, b.y),
                     __fmaf_rn(__fmul_rn(a.z, rstd), g.z, b.z), __fmaf_rn(__fmul_rn(a.w, rstd), g.w, b.w));
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

#endif  // __CUDACC__

}  // namespace dss
