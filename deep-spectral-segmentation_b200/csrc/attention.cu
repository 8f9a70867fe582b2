// Multi-head attention (head dim 64) on the Hopper tensor cores: O = softmax(Q K^T / 8) V, in both precision modes.
//
// Both kernels run one CTA per (128-query tile, head, image) with two warp groups, each owning 64 query rows. Thread 0
// drives the TMA: the Q tile once, the K_j / V_j tiles through a 2-stage ring shared by both warp groups (KvRing).
// Per key tile j, per warp group: S = Q K^T on wgmma into registers, the online softmax in registers (softmax_tile:
// row max / sum over the 4 lanes of a quad, base-2 exponent), P packed to fp16 in the register layout of the wgmma A
// operand (P never touches shared memory), O += P V on wgmma with A = P from registers and B = V (MN-major: keys x
// head dims). Keys past T are masked to -inf.
//
// attention_wgmma_kernel (DSS_VIT_PRECISION_FP16): Q / K / V come straight out of the packed qkv activations [B*T, 3d]
// (box 64 x 128, 128 B swizzle); 128-key tiles, S by wgmma m64 x 128 x 16 (x4), PV by m64 x 64 x 16 (x8); two CTAs per
// SM. The output leaves through the (then free) Q tile with one 3-D TMA store (rows past T clipped per image). Padding
// is not computed: an image's last key tile runs on the narrowest wgmma N of 8, 16, 32, 64, 96, 128 that covers its
// keys, and in an image's last query tile with at most 64 rows only warp group 0 runs.
//
// attention_split_kernel (DSS_VIT_PRECISION_FP32): fp32-equivalent accuracy on the fp16 tensor cores. Operands come
// from qkv_split_kernel (vit_kernels.cu), per head 192 columns of [B*T, 9d]:
//   Q' = [qhi | qhi/64 | 64 qlo]   K' = [khi | 64 klo | khi/64]   V' = [vhi | 64 vlo | vhi/64]
// so that S = Q' K'^T over K = 192 is qhi khi + qhi klo + qlo khi (12 k-steps), and with P = Phi + Plo split in registers
//   O += Phi Vhi + (Phi/64)(64 Vlo) + (64 Plo)(Vhi/64)          (three m64n64k16 passes of 4 k-steps per key tile)
// Softmax and the running row max / sum are fp32 (the row sum adds the unsplit fp32 p). Q' is 128 x 192 fp16 = 48 KB;
// a 128-key K'/V' stage would be 96 KB, so two stages would not fit beside Q' (240 KB > 227 KB). 64-key stages (K' and
// V' 24 KB each) give a two-stage ring in 144 KB: one CTA per SM, the next tile's load under the current tile's MMAs.
// The output (normalised O, split in A order, each group d wide, head h at columns h*64 of each group) is the proj
// GEMM's A operand and is stored straight from registers (rows past T skipped).
#include <math.h>

#include <type_traits>

#include "common.cuh"

namespace dss {

// mbarriers of an attention CTA: q_full (the Q tile landed) and, per stage s of the K/V ring, kv_full (the stage
// landed) and kv_empty (every warp group that runs the key loop is done with it)
template <int STAGES>
struct KvRing {
  uint32_t bar0;
  __device__ __forceinline__ uint32_t q_full() const { return bar0; }
  __device__ __forceinline__ uint32_t full(int s) const { return bar0 + 8u * (1 + s); }
  __device__ __forceinline__ uint32_t empty(int s) const { return bar0 + 8u * (1 + STAGES + s); }
  __device__ __forceinline__ void init(uint32_t groups) const {
    mbar_init(q_full(), 1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), groups);   // one arrival per warp group in the key loop
    }
    mbar_fence_init();
  }
  __device__ __forceinline__ void wait(int j) const {
    mbar_wait(full(j % STAGES), (j / STAGES) & 1);
    __syncwarp();   // wgmma is warp-aligned: reconverge after the per-thread barrier spin / thread 0's refill
  }
  // this warp group is done with K_j / V_j; thread 0 refills the slot with tile j + STAGES once every group in the key
  // loop is
  template <typename Load>
  __device__ __forceinline__ void release(int j, int nt, Load&& load_kv) const {
    const int s = j % STAGES;
    __syncwarp();
    if ((threadIdx.x & 127) == 0) mbar_arrive(empty(s));
    if (threadIdx.x == 0 && j + STAGES < nt) {
      mbar_wait(empty(s), (j / STAGES) & 1);
      load_kv(j + STAGES);
    }
  }
};

// softmax in base 2: p = 2^(s c - m c), c = log2(e) / sqrt(64)
constexpr float kSoftmaxScale = 1.4426950408889634f * 0.125f;

// One key tile of the online softmax: S holds NB 8-key blocks in the accumulator layout (sacc[4i], sacc[4i+1]: keys
// kbase + 8i + fc, +1 of row lane/4; sacc[4i+2], sacc[4i+3]: the same keys of row lane/4 + 8). Keys at or past T are
// masked, the running max m_run and sum l_run of both rows are updated, O is rescaled, and block i's probabilities go
// to pack(i, p0, p1, p2, p3) (p0, p1 of row lane/4; p2, p3 of row lane/4 + 8).
template <int NB, typename Pack>
__device__ __forceinline__ void softmax_tile(float (&sacc)[4 * NB], float (&o)[32], float (&m_run)[2], float (&l_run)[2],
                                             int kbase, int T, int fc, Pack&& pack) {
  const float sc = kSoftmaxScale;
  if (kbase + 8 * NB > T) {   // only the last tile can be partial
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      const int key = kbase + 8 * i + fc;
      if (key >= T) sacc[4 * i] = sacc[4 * i + 2] = -INFINITY;
      if (key + 1 >= T) sacc[4 * i + 1] = sacc[4 * i + 3] = -INFINITY;
    }
  }
  float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
  for (int i = 0; i < NB; ++i) {
    mx[0] = fmaxf(mx[0], fmaxf(sacc[4 * i], sacc[4 * i + 1]));
    mx[1] = fmaxf(mx[1], fmaxf(sacc[4 * i + 2], sacc[4 * i + 3]));
  }
  float corr[2], msc[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    corr[r] = ex2_approx((m_run[r] - mx[r]) * sc);   // first tile: 2^-inf = 0
    m_run[r] = mx[r];
    msc[r] = mx[r] * sc;
    l_run[r] *= corr[r];
  }
  float rs[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < NB; ++i) {
    const float p0 = ex2_approx(fmaf(sacc[4 * i], sc, -msc[0]));
    const float p1 = ex2_approx(fmaf(sacc[4 * i + 1], sc, -msc[0]));
    const float p2 = ex2_approx(fmaf(sacc[4 * i + 2], sc, -msc[1]));
    const float p3 = ex2_approx(fmaf(sacc[4 * i + 3], sc, -msc[1]));
    rs[0] += p0 + p1;
    rs[1] += p2 + p3;
    pack(i, p0, p1, p2, p3);
  }
  l_run[0] += rs[0];
  l_run[1] += rs[1];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    o[4 * i] *= corr[0]; o[4 * i + 1] *= corr[0];
    o[4 * i + 2] *= corr[1]; o[4 * i + 3] *= corr[1];
  }
}

// after the last tile: each row's sum across the 4 lanes of its quad
__device__ __forceinline__ void softmax_rowsum(float (&l_run)[2]) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
}

// Where a CTA's query tile lies: image b, its T token rows from row0(), the tile's first query q0(bm) of the image.
// A uniform batch of B images of T tokens: CTA (x, head, b) runs tile x of image b.
struct UniformTile {
  int b, T;
  __device__ __forceinline__ int q0(int bm) const { return blockIdx.x * bm; }
  __device__ __forceinline__ int row0() const { return b * T; }
};
// A ragged batch (vit.cu): CTA (x, head) runs tile x - tile_prefix[b] of the image b whose tiles
// [tile_prefix[b], tile_prefix[b + 1]) contain x.
struct RaggedTile {
  int b, T, first, tok_off;
  __device__ __forceinline__ RaggedTile(const RaggedImage* imgs, const int* tile_prefix, int B) {
    b = ragged_find(B, blockIdx.x, [&](int i) { return tile_prefix[i]; });
    first = tile_prefix[b];
    tok_off = imgs[b].tok_off;
    T = imgs[b].Hp * imgs[b].Wp + 1;
  }
  __device__ __forceinline__ int q0(int bm) const { return ((int)blockIdx.x - first) * bm; }
  __device__ __forceinline__ int row0() const { return tok_off; }
};

// ---------------------------------------------------------------------------------------------------------------
constexpr int FA_BM = 128, FA_BN = 128, FA_D = 64, FA_THREADS = 256;
constexpr int FA_TILE = FA_BM * FA_D * 2;             // 16 KB: one [128 x 64] fp16 tile
constexpr int FA_KV_STAGES = 2;
// Q (reused as the output box) | K ring | V ring = 80 KB: two CTAs per SM
constexpr int FA_SMEM = FA_TILE * (1 + 2 * FA_KV_STAGES) + 1024;

// One CTA: the query tile `loc` names, head blockIdx.y. RAGGED (packed images of different sizes): tmO is the 2D output
// [rows, d]; an image's last tile, if it ends past T, is stored from registers row by row, so it writes no row of the
// next image; `out` is that output.
template <bool RAGGED, typename Loc>
__device__ __forceinline__ void attention_wgmma_tile(const CUtensorMap& tmQKV, const CUtensorMap& tmO, Loc loc,
                                                     int heads, __half* out) {
  extern __shared__ uint8_t fa_smem[];
  __shared__ __align__(8) uint64_t bars[1 + 2 * FA_KV_STAGES];
  const uint32_t raw = smem_u32(fa_smem);
  const uint32_t base = (raw + 1023u) & ~1023u;   // the 128 B swizzle pattern is a function of address bits [7,10)
  const uint32_t sQ = base, sK = base + FA_TILE, sV = sK + FA_KV_STAGES * FA_TILE;
  const KvRing<FA_KV_STAGES> ring{smem_u32(bars)};

  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = tid >> 7, wi = (tid >> 5) & 3;
  const int q0 = loc.q0(FA_BM), h = blockIdx.y, b = loc.b;
  const int d = heads * FA_D;
  const int T = loc.T;
  const int nt = (T + FA_BN - 1) / FA_BN;
  const int row0 = loc.row0();   // first row of this image in [rows, 3d]
  // a tile with at most 64 query rows (an image's last) leaves warp group 1 without rows: it skips the key loop
  const int groups = q0 + 64 >= T ? 1 : 2;

  auto load_kv = [&](int j) {
    const int s = j % FA_KV_STAGES;
    mbar_arrive_expect_tx(ring.full(s), 2 * FA_TILE);
    tma_load_2d(sK + s * FA_TILE, &tmQKV, ring.full(s), d + h * FA_D, row0 + j * FA_BN);
    tma_load_2d(sV + s * FA_TILE, &tmQKV, ring.full(s), 2 * d + h * FA_D, row0 + j * FA_BN);
  };
  if (tid == 0) {
    tma_prefetch_desc(&tmQKV);
    tma_prefetch_desc(&tmO);
    ring.init(groups);
    mbar_arrive_expect_tx(ring.q_full(), FA_TILE);
    tma_load_2d(sQ, &tmQKV, ring.q_full(), h * FA_D, row0 + q0);
    for (int j = 0; j < FA_KV_STAGES && j < nt; ++j) load_kv(j);
  }
  __syncthreads();

  const int fc = 2 * (lane & 3);                    // column of this thread inside an 8-column block
  float m_run[2] = {-INFINITY, -INFINITY};           // rows lane/4 and lane/4 + 8 of this warp's 16
  float l_run[2] = {0.f, 0.f};
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  const uint64_t qdesc0 = wgmma_desc_sw128(sQ + wg * 64 * 128);

  // Key tile j with NB 8-key blocks (keys 128 j + [0, 8 NB)): S on wgmma m64 x 8NB x 16 (x4), the softmax, then
  // O += P V over ceil(NB / 2) 16-key steps. A narrower tile gives the same bits as the full one: each S element is the
  // same four k16 products, and the keys it drops are past T, so they would only add -inf to the row max, 0 to the row
  // sum and exact zeros (P = 0 times finite V rows) to O.
  auto key_tile = [&](int j, auto nb) {
    constexpr int NB = decltype(nb)::value, KS = (NB + 1) / 2;
    const int s = j % FA_KV_STAGES;
    ring.wait(j);
    float sacc[4 * NB];
    // opaque per tile, so that the compiler does not hoist the k-step descriptors out of the key loop (and spill them)
    uint64_t qdesc = qdesc0;
    asm volatile("" : "+l"(qdesc));
    const uint64_t kdesc = wgmma_desc_sw128(sK + s * FA_TILE);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < FA_D / 16; ++k) Wgmma<8 * NB>::ss(sacc, qdesc + 2u * k, kdesc + 2u * k, k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(sacc);
    // accumulator layout of two adjacent 8-key blocks == register A-operand layout of one 16-key step
    uint32_t pf[KS][4];
    if constexpr (NB % 2) pf[KS - 1][2] = pf[KS - 1][3] = 0u;   // the missing block of the last step: P = 0
    softmax_tile<NB>(sacc, o, m_run, l_run, j * FA_BN, T, fc, [&](int i, float p0, float p1, float p2, float p3) {
      pf[i >> 1][(i & 1) * 2 + 0] = pack_half2(p0, p1);
      pf[i >> 1][(i & 1) * 2 + 1] = pack_half2(p2, p3);
    });
    const uint64_t vdesc = wgmma_desc_sw128(sV + s * FA_TILE);   // +16 key rows = +2048 B
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) wgmma_m64n64_rs_tb(o, pf[ks], vdesc + 128u * ks);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(o);
    ring.release(j, nt, load_kv);
  };
  if (wg < groups) {
    mbar_wait(ring.q_full(), 0);
    __syncwarp();
    for (int j = 0; j < nt - 1; ++j) key_tile(j, std::integral_constant<int, 16>{});
    // the last key tile holds T - 128 (nt - 1) keys: the narrowest of 8, 16, 32, 64, 96 or 128 keys that covers them
    const int r = T - FA_BN * (nt - 1);
    if (r <= 8)
      key_tile(nt - 1, std::integral_constant<int, 1>{});
    else if (r <= 16)
      key_tile(nt - 1, std::integral_constant<int, 2>{});
    else if (r <= 32)
      key_tile(nt - 1, std::integral_constant<int, 4>{});
    else if (r <= 64)
      key_tile(nt - 1, std::integral_constant<int, 8>{});
    else if (r <= 96)
      key_tile(nt - 1, std::integral_constant<int, 12>{});
    else
      key_tile(nt - 1, std::integral_constant<int, 16>{});
  }

  // finalise: normalise, fp16 into this group's half of the Q tile (swizzled as the output box), one TMA store of the
  // 128 x 64 box. A group without rows stores nothing: the ragged partial tile skips rows >= T, and the uniform box
  // store clips them.
  softmax_rowsum(l_run);
  const float inv0 = 1.0f / l_run[0], inv1 = 1.0f / l_run[1];
  const int r0 = 64 * wg + 16 * wi + (lane >> 2);
  if constexpr (RAGGED) {
    if (q0 + FA_BM > T) {   // the image's last, partial tile: masked direct stores
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = q0 + r0 + 8 * hh;
        if (row >= T) continue;
        const float inv = hh ? inv1 : inv0;
        uint32_t* orow = reinterpret_cast<uint32_t*>(out + ((long long)row0 + row) * d + h * FA_D + fc);
#pragma unroll
        for (int i = 0; i < 8; ++i) orow[4 * i] = pack_half2(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv);
      }
      return;
    }
  }
  if (wg < groups) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = r0 + 8 * hh;
        const float inv = hh ? inv1 : inv0;
        const uint32_t addr = sw128_addr(sQ, row, i) + (lane & 3) * 4;
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr),
                     "r"(pack_half2(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv))
                     : "memory");
      }
    }
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (tid == 0) {
    if constexpr (RAGGED)
      tma_store_2d(&tmO, sQ, h * FA_D, row0 + q0);
    else
      tma_store_3d(&tmO, sQ, h * FA_D, q0, b);
    tma_store_commit();
    tma_store_wait_all<0>();
  }
}

__global__ void __launch_bounds__(FA_THREADS, 2)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmO, int T,
                       int heads) {
  attention_wgmma_tile<false>(tmQKV, tmO, UniformTile{(int)blockIdx.z, T}, heads, nullptr);
}

__global__ void __launch_bounds__(FA_THREADS, 2)
attention_wgmma_ragged_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmO,
                              const RaggedImage* __restrict__ imgs, const int* __restrict__ tile_prefix, int B,
                              int heads, __half* __restrict__ out) {
  attention_wgmma_tile<true>(tmQKV, tmO, RaggedTile(imgs, tile_prefix, B), heads, out);
}

// ---------------------------------------------------------------------------------------------------------------
constexpr int AS_BM = 128, AS_BN = 64, AS_THREADS = 256, AS_STAGES = 2;
constexpr int AS_BOX = 64 * 64 * 2;                    // 8 KB: one 64-row x 64-column fp16 TMA box
constexpr int AS_Q = 3 * 2 * AS_BOX;                   // Q': 3 groups x 128 rows
constexpr int AS_KV = 3 * AS_BOX;                      // one K' or V' stage: 3 groups x 64 keys
constexpr int AS_SMEM = AS_Q + 2 * AS_STAGES * AS_KV + 1024;

// One CTA: the query tile `loc` names, head blockIdx.y (rows past T are not stored).
template <typename Loc>
__device__ __forceinline__ void attention_split_tile(const CUtensorMap& tmQKV, __half* __restrict__ out, Loc loc,
                                                     int heads) {
  extern __shared__ uint8_t as_smem[];
  __shared__ __align__(8) uint64_t bars[1 + 2 * AS_STAGES];
  const uint32_t base = (smem_u32(as_smem) + 1023u) & ~1023u;
  const uint32_t sQ = base, sK = base + AS_Q, sV = sK + AS_STAGES * AS_KV;
  const KvRing<AS_STAGES> ring{smem_u32(bars)};

  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = tid >> 7, wi = (tid >> 5) & 3;
  const int q0 = loc.q0(AS_BM), h = blockIdx.y;
  const int d = heads * 64;
  const int T = loc.T;
  const int nt = (T + AS_BN - 1) / AS_BN;
  const int row0 = loc.row0();

  auto load_kv = [&](int j) {
    const int s = j % AS_STAGES;
    mbar_arrive_expect_tx(ring.full(s), 2 * AS_KV);
    for (int g = 0; g < 3; ++g) {
      tma_load_2d(sK + s * AS_KV + g * AS_BOX, &tmQKV, ring.full(s), 3 * d + h * 192 + g * 64, row0 + j * AS_BN);
      tma_load_2d(sV + s * AS_KV + g * AS_BOX, &tmQKV, ring.full(s), 6 * d + h * 192 + g * 64, row0 + j * AS_BN);
    }
  };
  if (tid == 0) {
    tma_prefetch_desc(&tmQKV);
    ring.init(2);
    mbar_arrive_expect_tx(ring.q_full(), AS_Q);
    // Q' group g: rows 0-63 at +0, rows 64-127 at +8 KB, so each group is one 128-row swizzled tile
    for (int g = 0; g < 3; ++g)
      for (int half = 0; half < 2; ++half)
        tma_load_2d(sQ + (2 * g + half) * AS_BOX, &tmQKV, ring.q_full(), h * 192 + g * 64, row0 + q0 + 64 * half);
    for (int j = 0; j < AS_STAGES && j < nt; ++j) load_kv(j);
  }
  __syncthreads();

  const int fc = 2 * (lane & 3);
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  mbar_wait(ring.q_full(), 0);
  __syncwarp();

  for (int j = 0; j < nt; ++j) {
    const int s = j % AS_STAGES;
    ring.wait(j);
    float sacc[32];
    wgmma_fence();
#pragma unroll
    for (int g = 0; g < 3; ++g) {
      const uint64_t qdesc = wgmma_desc_sw128(sQ + 2 * g * AS_BOX + wg * AS_BOX);
      const uint64_t kdesc = wgmma_desc_sw128(sK + s * AS_KV + g * AS_BOX);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64_ss(sacc, qdesc + 2u * k, kdesc + 2u * k, (g | k) != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(sacc);
    // P in the register A-operand layout (two adjacent 8-key blocks = one 16-key step), split into its three groups
    uint32_t p_hi[4][4], p_his[4][4], p_los[4][4];
    softmax_tile<8>(sacc, o, m_run, l_run, j * AS_BN, T, fc, [&](int i, float p0, float p1, float p2, float p3) {
      const SplitF16 sp[4] = {split_f16(p0), split_f16(p1), split_f16(p2), split_f16(p3)};
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        p_hi[i >> 1][(i & 1) * 2 + r] = pack_h2(sp[2 * r].hi, sp[2 * r + 1].hi);
        p_his[i >> 1][(i & 1) * 2 + r] = pack_h2(sp[2 * r].hi_s, sp[2 * r + 1].hi_s);
        p_los[i >> 1][(i & 1) * 2 + r] = pack_h2(sp[2 * r].lo_s, sp[2 * r + 1].lo_s);
      }
    });
    // V' group g tile: 64 keys x 64 head dims, MN-major; +16 keys = +2048 B
    const uint64_t v_hi = wgmma_desc_sw128(sV + s * AS_KV), v_los = wgmma_desc_sw128(sV + s * AS_KV + AS_BOX),
                   v_his = wgmma_desc_sw128(sV + s * AS_KV + 2 * AS_BOX);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < AS_BN / 16; ++ks) wgmma_m64n64_rs_tb(o, p_hi[ks], v_hi + 128u * ks);
#pragma unroll
    for (int ks = 0; ks < AS_BN / 16; ++ks) wgmma_m64n64_rs_tb(o, p_his[ks], v_los + 128u * ks);
#pragma unroll
    for (int ks = 0; ks < AS_BN / 16; ++ks) wgmma_m64n64_rs_tb(o, p_los[ks], v_his + 128u * ks);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(o);
    ring.release(j, nt, load_kv);
  }

  softmax_rowsum(l_run);
  const float inv[2] = {1.0f / l_run[0], 1.0f / l_run[1]};
  const int r0 = q0 + 64 * wg + 16 * wi + (lane >> 2);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = r0 + 8 * hh;
    if (row >= T) continue;
    __half* orow = out + ((long long)row0 + row) * 3 * d + h * 64 + fc;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const SplitF16 a = split_f16(o[4 * i + 2 * hh] * inv[hh]);
      const SplitF16 c = split_f16(o[4 * i + 2 * hh + 1] * inv[hh]);
      store_split(reinterpret_cast<uint32_t*>(orow + 8 * i), d / 2, 0, pack_h2(a.hi, c.hi), pack_h2(a.hi_s, c.hi_s),
                  pack_h2(a.lo_s, c.lo_s));
    }
  }
}

__global__ void __launch_bounds__(AS_THREADS, 1)
attention_split_kernel(const __grid_constant__ CUtensorMap tmQKV, __half* __restrict__ out, int T, int heads) {
  attention_split_tile(tmQKV, out, UniformTile{(int)blockIdx.z, T}, heads);
}

__global__ void __launch_bounds__(AS_THREADS, 1)
attention_split_ragged_kernel(const __grid_constant__ CUtensorMap tmQKV, __half* __restrict__ out,
                              const RaggedImage* __restrict__ imgs, const int* __restrict__ tile_prefix, int B,
                              int heads) {
  attention_split_tile(tmQKV, out, RaggedTile(imgs, tile_prefix, B), heads);
}

// ---------------------------------------------------------------------------------------------------------------
int launch_attention_tc(const void* qkv, void* out, int B, int T, int heads, cudaStream_t st) {
  DSS_REQUIRE(B > 0 && T > 0 && heads > 0, "attention: empty problem");
  static bool attr_set = false;
  if (!attr_set) {
    DSS_CHECK_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FA_SMEM));
    attr_set = true;
  }
  CUtensorMap tm, tmO;
  int rc = make_tmap_f16(&tm, qkv, B * T, 3 * heads * FA_D, FA_BM);
  if (rc) return rc;
  if ((rc = make_tmap_out3d_f16(&tmO, out, B, T, heads * FA_D))) return rc;
  dim3 grid(cdiv(T, FA_BM), heads, B);
  LaunchScope scope(st, KC_ATTENTION);
  attention_wgmma_kernel<<<grid, FA_THREADS, FA_SMEM, st>>>(tm, tmO, T, heads);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

// qkv_split [B*T, 9d] (qkv_split_kernel's layout) -> out [B*T, 3d] split attention output
int launch_attention_split(const void* qkv_split, void* out, int B, int T, int heads, cudaStream_t st) {
  DSS_REQUIRE(qkv_split && out, "attention_split: null pointer");
  DSS_REQUIRE(B > 0 && T > 0 && heads > 0, "attention_split: empty problem");
  static bool attr_set = false;
  if (!attr_set) {
    DSS_CHECK_CUDA(cudaFuncSetAttribute(attention_split_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AS_SMEM));
    attr_set = true;
  }
  CUtensorMap tm;
  int rc = make_tmap_f16(&tm, qkv_split, B * T, 9 * heads * 64, 64);
  if (rc) return rc;
  dim3 grid(cdiv(T, AS_BM), heads, B);
  LaunchScope scope(st, KC_ATTENTION);
  attention_split_kernel<<<grid, AS_THREADS, AS_SMEM, st>>>(tm, reinterpret_cast<__half*>(out), T, heads);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_attention_tc_ragged(const void* qkv, void* out, const RaggedImage* imgs, const int* tile_prefix, int B,
                               long long M, int tiles, int heads, cudaStream_t st) {
  DSS_REQUIRE(B > 0 && M > 0 && tiles > 0 && heads > 0, "attention_ragged: empty problem");
  static bool attr_set = false;
  if (!attr_set) {
    DSS_CHECK_CUDA(cudaFuncSetAttribute(attention_wgmma_ragged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        FA_SMEM));
    attr_set = true;
  }
  CUtensorMap tm, tmO;
  int rc = make_tmap_f16(&tm, qkv, (int)M, 3 * heads * FA_D, FA_BM);
  if (rc) return rc;
  if ((rc = make_tmap_out(&tmO, out, (int)M, heads * FA_D, 0))) return rc;
  LaunchScope scope(st, KC_ATTENTION);
  attention_wgmma_ragged_kernel<<<dim3(tiles, heads), FA_THREADS, FA_SMEM, st>>>(tm, tmO, imgs, tile_prefix, B, heads,
                                                                                 reinterpret_cast<__half*>(out));
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

int launch_attention_split_ragged(const void* qkv_split, void* out, const RaggedImage* imgs, const int* tile_prefix,
                                  int B, long long M, int tiles, int heads, cudaStream_t st) {
  DSS_REQUIRE(B > 0 && M > 0 && tiles > 0 && heads > 0, "attention_split_ragged: empty problem");
  static bool attr_set = false;
  if (!attr_set) {
    DSS_CHECK_CUDA(cudaFuncSetAttribute(attention_split_ragged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        AS_SMEM));
    attr_set = true;
  }
  CUtensorMap tm;
  int rc = make_tmap_f16(&tm, qkv_split, (int)M, 9 * heads * 64, 64);
  if (rc) return rc;
  LaunchScope scope(st, KC_ATTENTION);
  attention_split_ragged_kernel<<<dim3(tiles, heads), AS_THREADS, AS_SMEM, st>>>(tm, reinterpret_cast<__half*>(out),
                                                                                 imgs, tile_prefix, B, heads);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

}  // namespace dss

extern "C" int dss_op_attention_tc_f16(const void* qkv, void* out, int B, int T, int heads, dss_stream_t stream) {
  return dss::launch_attention_tc(qkv, out, B, T, heads, static_cast<cudaStream_t>(stream));
}

extern "C" int dss_op_attention_split_f16(const float* qkv, void* qkv_split, void* out, int B, int T, int heads,
                                          dss_stream_t stream) {
  DSS_REQUIRE(qkv, "attention_split: null pointer");
  DSS_REQUIRE(B > 0 && T > 0 && heads > 0, "attention_split: empty problem");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = dss::launch_qkv_split(qkv, qkv_split, (long long)B * T, heads * 64, st);
  if (rc) return rc;
  return dss::launch_attention_split(qkv_split, out, B, T, heads, st);
}
