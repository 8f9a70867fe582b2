// out = epilogue(A[M,K] * Wt[N,K]^T + bias) with fp16 operands, fp32 accumulation in registers (Hopper wgmma).
//
// Persistent kernel, one CTA per SM, 128 x BN output tiles handed out round-robin (n fastest, so CTAs that run
// together share the A rows in L2 and the whole weight matrix stays L2-resident):
//   warp group 0     : TMA producer (one warp: cp.async.bulk.tensor 2D, 128B swizzle, 64-wide K slabs); the ring keeps
//                      running across tile boundaries, so loads for the next tile are in flight during the epilogue.
//                      It gives most of its registers to the MMA groups (setmaxnreg).
//   warp groups 1, 2 : wgmma m64 x BN x 16 on 64 rows each of the tile (both operands straight from the swizzled
//                      slabs), then the epilogue from the register accumulators: +bias / exact-erf GELU -> 128 B-swizzled
//                      staging box -> TMA store (or TMA reduce-add for the residual)
// CTAs run as CLUSTERS OF TWO that work on vertically adjacent tiles (same n, m and m+1): each CTA fetches half of
// the weight tile and TMA-multicasts it into both CTAs' shared memory, which halves the L2 -> SM traffic of the weight
// operand. A slab is free once the MMA groups of both CTAs have retired their wgmmas on it.
// Both operands are K-major, which is the native layout of activations [rows, features] and of torch Linear
// weights [out, in]; no transposes anywhere.
//
// Two schedules share the producer and the cluster / ring protocol:
//   cooperative (gemm_f16_wgmma_kernel): both MMA groups work on the same 128 x BN tile, each on 64 of its rows, so the
//     tensor cores idle while the tile's epilogue runs. Used by the row-remapping epilogues, the affinity GEMM (whose
//     symmetric mode keeps the CTA pair in lock step) and dss_debug_gemm_cfg.
//   ping-pong (gemm_f16_pingpong_kernel): each MMA group owns whole 128 x 128 tiles and the two groups take alternate
//     work items; a pair of named barriers hands the "MMA turn" from one group to the other, so one group's epilogue
//     runs under the other group's wgmmas. Used by the four ViT epilogues (qkv, proj, fc1, fc2).
#include <math.h>

#include "gemm_pipeline.cuh"

namespace dss {

constexpr int BM = 128;
constexpr int A_ATOM_BYTES = BM * BK * 2;
constexpr int CONSUMER_WGS = 2;                 // MMA + epilogue warp groups, each owns 64 rows of the 128-row tile
constexpr int EPI_THREADS = CONSUMER_WGS * 128;
constexpr int GEMM_THREADS = 128 + EPI_THREADS; // warp group 0: TMA producer (one warp issues, three idle)
constexpr int STG_LD = 36;               // manual path staging chunk: 128 rows x 32 cols fp32, row pitch 36
constexpr int STG_BYTES = BM * STG_LD * 4;
constexpr int BOX_BYTES = BM * 128;      // TMA-store path staging box: 128 rows x 128 bytes (swizzled)

// epilogues whose output rows are the GEMM rows: written with TMA (the row-remapping ones keep the manual path)
constexpr int EPI_AFFINITY_F32 = 100;    // internal epilogue id (not in the public enum): batched patch-affinity tile
// internal ids of the ragged ViT batch: DSS_EPI_PATCH_F32 / DSS_EPI_DROPCLS_F32 with the destination row of GEMM row m
// read from p.row_map[m] (-1: skip) instead of computed from rin / rout; the patch epilogue's positional row is that
// destination row of p.aux (laid out like the residual stream)
constexpr int EPI_PATCH_ROWS_F32 = 101, EPI_DROPCLS_ROWS_F32 = 102;
__host__ __device__ constexpr bool epi_uses_tma_store(int epi) {
  return epi == DSS_EPI_BIAS_F16 || epi == DSS_EPI_BIAS_GELU_F16 || epi == DSS_EPI_BIAS_RESID_F32 ||
         epi == DSS_EPI_BIAS_F32 || epi == EPI_AFFINITY_F32;
}
// Ring stage = one 64-deep K slab of A (128 rows) and B (BN rows); as many stages as the shared-memory budget leaves
// next to the output staging (at most 6).
// Ping-pong (PP): 32 KB stages of 128 x 128 tiles next to two double-buffered 16 KB boxes per group = 5 stages
// (6 * 32 + 4 * 16 KB would not fit). Double buffering keeps a group's store of one box under its writes of the next.
template <int EPI, int BN, bool PP = false> struct TileCfg {
  static constexpr int B_ATOM_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_ATOM_BYTES + B_ATOM_BYTES;   // [A slab | B slab]
  // TMA path: two swizzled output boxes (+ the affinity epilogue's row-major fp32 copy of one box), two per consumer
  // warp group for the ping-pong schedule; manual path: two fp32 chunks
  static constexpr int STAGING_BYTES = PP ? CONSUMER_WGS * 2 * BOX_BYTES
                                     : epi_uses_tma_store(EPI) ? 2 * BOX_BYTES + (EPI == EPI_AFFINITY_F32 ? STG_BYTES : 0)
                                                               : 2 * STG_BYTES;
  static constexpr int MAX_STAGES = (SMEM_BUDGET - 1024 - 256 - STAGING_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = MAX_STAGES > 6 ? 6 : MAX_STAGES;
  // ring | staging | barriers | alignment slack
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + 256 + 1024;
  static_assert(STAGES >= 2, "shared memory budget");
};
// Ping-pong tile: 128 x 128 per consumer warp group, two m64n128k16 per k-step (128 accumulator registers per thread)
constexpr int PP_BN = 128;
static_assert(TileCfg<DSS_EPI_BIAS_F16, PP_BN, true>::STAGES == 5, "ping-pong ring depth");


struct EpiParams {
  void* out;
  const float* bias;
  const float* aux;
  int ldo;
  int rin, rout;
  // batched mode (gridDim.z = images): operand rows of image z start at z * batch_rows
  int batch_rows;
  // affinity epilogue
  const unsigned int* img_max;  // [images] float bits of max(W) per image
  const unsigned int* img_absmax;  // [images] float bits of max|f| when the features were pre-scaled by 2^-e (else null)
  const uint8_t* counts;        // [images, M, M] colour-KNN counts or null
  float lambda;
  int threshold;                // bit 0: relu threshold, bit 1: do not divide by max(W)
  int perm_blocks;              // B operand K-slab permutation for the split-fp16 Gram product (0 = none)
  // symmetric (affinity) mode: only tiles on or above the diagonal are computed; each strictly-upper tile is also
  // stored transposed, and per-tile row / column sums go to deg_part [images, 2 * 4 * tiles, ld_part] (degree fusion)
  int tri;
  float* deg_part;
  int ld_part;
  // phase trace (dss_debug_gemm_trace / dss_debug_affinity_trace only; read by the TRACE instantiations, layout at
  // trace_stride)
  unsigned long long* trace;
  // destination row per GEMM row (EPI_PATCH_ROWS_F32 / EPI_DROPCLS_ROWS_F32)
  const int* row_map;
};

// Phase trace layout, per CTA (blockIdx.x): [0] ns the producer warp spent waiting on empty ring slots, [1..3] unused,
// then for consumer warp group w and the j-th tile that group ran, four %globaltimer stamps at 4 + 4 * (w * tmax + j):
// tile start (for the ping-pong schedule: once the group holds the MMA turn), first full-barrier wait satisfied, last
// wgmma retired (wgmma_wait<0>), epilogue issued. tmax = cdiv(work items, clusters) bounds the tiles of one CTA.
__host__ __device__ constexpr long long trace_stride(int total_items, int clusters) {
  return 4 + 8ll * ((total_items + clusters - 1) / clusters);
}

// Row of the output buffer that GEMM row m maps to (or -1: skip).
template <int EPI>
__device__ __forceinline__ long long out_row(int m, const EpiParams& p) {
  if constexpr (EPI == DSS_EPI_PATCH_F32) {
    return (long long)(m / p.rin) * p.rout + (m % p.rin) + 1;
  } else if constexpr (EPI == DSS_EPI_DROPCLS_F32) {
    const int t = m % p.rin;
    return t == 0 ? -1 : (long long)(m / p.rin) * p.rout + t - 1;
  } else if constexpr (EPI == EPI_PATCH_ROWS_F32 || EPI == EPI_DROPCLS_ROWS_F32) {
    return __ldg(p.row_map + m);
  } else {
    return m;
  }
}

// Applies the epilogue to 32 consecutive columns [n, n+32) of one row and stores them.
// ---- coalesced epilogue, second phase: one warp owns one output row of the tile at a time, lane l owns columns
// n..n+3 (n = n0 + 4*l), so every global access of a warp is one contiguous 512 B (fp32) / 256 B (fp16) segment.
template <int EPI>
__device__ __forceinline__ void store_row4(float4 v, int m, int n, const EpiParams& p) {
  const long long r = out_row<EPI>(m, p);
  if (r < 0) return;
  if constexpr (EPI == DSS_EPI_BIAS_F16 || EPI == DSS_EPI_BIAS_GELU_F16) {
    uint2 q;
    q.x = pack_half2(v.x, v.y);
    q.y = pack_half2(v.z, v.w);
    *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(p.out) + r * p.ldo + n) = q;
  } else {
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + r * p.ldo + n) = v;
  }
}

// ---- one thread = one row x 32 columns (used by the CUDA-core checker kernel only)
template <int EPI>
__device__ __forceinline__ void epilogue_store(const float (&v)[32], int m, int n, const EpiParams& p) {
#pragma unroll
  for (int j = 0; j < 32; j += 4) {
    float4 x = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
    if constexpr (EPI == DSS_EPI_BIAS_GELU_F16) {
      x.x = gelu_erf(x.x); x.y = gelu_erf(x.y); x.z = gelu_erf(x.z); x.w = gelu_erf(x.w);
    }
    if constexpr (EPI == DSS_EPI_BIAS_RESID_F32) {
      const float4 y = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.out) + (long long)m * p.ldo + n + j);
      x.x += y.x; x.y += y.y; x.z += y.z; x.w += y.w;
    }
    if constexpr (EPI == DSS_EPI_PATCH_F32) {
      const float4 y = __ldg(reinterpret_cast<const float4*>(p.aux + (long long)((m % p.rin) + 1) * p.ldo + n + j));
      x.x += y.x; x.y += y.y; x.z += y.z; x.w += y.w;
    }
    store_row4<EPI>(x, m, n + j, p);
  }
}

struct TileCoord { int m0, n0, z; };
// work item t of a cluster = (image z, pair of vertically adjacent m-tiles, n-tile); CTA `rank` takes tile 2*pair+rank
template <int BN>
__device__ __forceinline__ TileCoord decode_tile(int t, int pairs_m, int tiles_n, int rank, int tri = 0) {
  if (tri) {
    // symmetric output (BN == BM): row pair p only visits n-tiles j >= 2p. Tile (2p+1, 2p) of the odd CTA lies below the
    // diagonal: its slabs are waited for and released (the pair runs in lock step on the shared B tile), but no wgmma
    // is issued for it and nothing is stored.
    int per_img = 0;
    for (int p = 0; p < pairs_m; ++p) per_img += max(tiles_n - 2 * p, 0);
    const int z = t / per_img;
    int rem = t - z * per_img, p = 0;
    for (; p < pairs_m; ++p) {
      const int cnt = max(tiles_n - 2 * p, 0);
      if (rem < cnt) break;
      rem -= cnt;
    }
    return TileCoord{(2 * p + rank) * BM, (2 * p + rem) * BN, z};
  }
  const int per_img = pairs_m * tiles_n;
  const int z = t / per_img, rem = t - z * per_img;
  return TileCoord{((rem / tiles_n) * 2 + rank) * BM, (rem % tiles_n) * BN, z};
}

// The k-steps of one slab on the first w columns of a 128-wide tile, w in {0, 8, 16, 32, 64, 96, 128} (0: no wgmma).
// The accumulators of a narrow wgmma are a prefix of the wide one's, and each output element is the same four k16
// products whatever the width; the registers past the prefix keep stale values.
__device__ __forceinline__ void mma_slab_cols(float (&acc)[64], int w, uint64_t adesc, uint64_t bdesc, bool first) {
  switch (w) {
    case 8: mma_slab<8>(*reinterpret_cast<float (*)[4]>(&acc), adesc, bdesc, first); break;
    case 16: mma_slab<16>(*reinterpret_cast<float (*)[8]>(&acc), adesc, bdesc, first); break;
    case 32: mma_slab<32>(*reinterpret_cast<float (*)[16]>(&acc), adesc, bdesc, first); break;
    case 64: mma_slab<64>(*reinterpret_cast<float (*)[32]>(&acc), adesc, bdesc, first); break;
    case 96: mma_slab<96>(*reinterpret_cast<float (*)[48]>(&acc), adesc, bdesc, first); break;
    case 128: mma_slab<128>(acc, adesc, bdesc, first); break;
  }
}
// Narrowest of those widths that covers r >= 1 columns
__device__ __forceinline__ int mma_cols(int r) {
  return r <= 8 ? 8 : r <= 16 ? 16 : r <= 32 ? 32 : r <= 64 ? 64 : r <= 96 ? 96 : 128;
}

// Accumulator fragment helpers. Warp group wg, warp wi (0..3 inside the group), lane l hold for each 8-column block i
// of the tile: acc[4i], acc[4i+1] = row 64 wg + 16 wi + l/4, columns 8i + 2(l%4) + {0,1}; acc[4i+2], acc[4i+3] = the
// same columns 8 rows further down.
__device__ __forceinline__ int frag_row(int wg, int wi, int lane) { return 64 * wg + 16 * wi + (lane >> 2); }

// TMA producer (warp 0 of warp group 0) of both schedules: the CTA's work items in order, one ring slot per 64-deep K
// slab, the ring position carried across tiles. The whole warp runs the loop with warp-uniform values; one elected
// lane issues. The slab a slot held is free once one consumer group of EACH CTA has released it (empty barrier).
template <int BN, int STAGES, int STAGE_BYTES, bool TRACE>
__device__ __forceinline__ void produce(const CUtensorMap* tmA, const CUtensorMap* tmB, uint32_t base,
                                        const RingBars<STAGES>& bars, int num_kb, int cid, int ncl, int rank,
                                        int pairs_m, int tiles_n, int total_items, const EpiParams& p) {
  constexpr int B_ATOM_BYTES = BN * BK * 2;
  const int lane = threadIdx.x & 31;
  const uint32_t ubase = __shfl_sync(0xffffffffu, base, 0);
  [[maybe_unused]] unsigned long long waited = 0;
  RingPos<STAGES> pos;   // carried across tiles
  for (int t = cid; t < total_items; t += ncl) {
    const TileCoord tc = decode_tile<BN>(t, pairs_m, tiles_n, rank, p.tri);
    const int row_base = tc.z * p.batch_rows;
    for (int kb = 0; kb < num_kb; ++kb) {
      [[maybe_unused]] unsigned long long t0;
      if constexpr (TRACE) t0 = globaltimer();
      mbar_wait(bars.empty(pos.slot), pos.phase ^ 1u);
      if constexpr (TRACE) waited += globaltimer() - t0;
      const uint32_t sa = ubase + pos.slot * STAGE_BYTES;
      const uint32_t fb = bars.full(pos.slot);
      // split-fp16 Gram product: A = [hi | hi/64 | 64 lo], B = [hi | 64 lo | hi/64] are the same array read with the
      // last two groups of K slabs swapped
      int kbB = kb;
      if (p.perm_blocks > 0 && kb >= p.perm_blocks && kb < 3 * p.perm_blocks)
        kbB = kb < 2 * p.perm_blocks ? kb + p.perm_blocks : kb - p.perm_blocks;
      if (elect_one()) {
        mbar_arrive_expect_tx(fb, STAGE_BYTES);
        tma_load_2d(sa, tmA, fb, kb * BK, row_base + tc.m0);
        // this CTA's half of the weight slab (box 64 x BN/2 rows), delivered to both CTAs of the pair
        tma_load_2d_mc(sa + A_ATOM_BYTES + rank * (B_ATOM_BYTES / 2), tmB, fb, kbB * BK,
                       row_base + tc.n0 + rank * (BN / 2), (uint16_t)0x3);
      }
      __syncwarp();
      pos.advance();
    }
  }
  if constexpr (TRACE) {
    if (lane == 0) p.trace[blockIdx.x * trace_stride(total_items, ncl)] = waited;
  }
}

template <int EPI, int BN, bool TRACE = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_f16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const __grid_constant__ CUtensorMap tmC, int M, int N, int K, int pairs_m, int tiles_n,
                      int total_items, EpiParams p) {
  static_assert(!TRACE || epi_uses_tma_store(EPI), "traced: the TMA-store epilogues only");
  using Cfg = TileCfg<EPI, BN>;
  constexpr int STAGES = Cfg::STAGES, STAGE_BYTES = Cfg::STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024 B alignment (the swizzle pattern is a function of address bits [7,10))
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - raw);
  float* stage_base = reinterpret_cast<float*>(gbase + STAGES * STAGE_BYTES);
  const RingBars<STAGES> bars{base + STAGES * STAGE_BYTES + Cfg::STAGING_BYTES};

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_kb = (K + BK - 1) / BK;
  const int rank = (int)cluster_ctarank();          // 0 / 1 inside the CTA pair
  const int cid = blockIdx.x >> 1, ncl = gridDim.x >> 1;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if constexpr (epi_uses_tma_store(EPI)) tma_prefetch_desc(&tmC);
    // released by the MMA warp groups of BOTH CTAs (each CTA's producer writes half of the B slab into the other)
    bars.init(2 * CONSUMER_WGS);
    mbar_fence_init();
  }
  __syncthreads();
  cluster_sync_all();   // both CTAs' barriers are initialised before any remote arrive / multicast can reach them

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0)
      produce<BN, STAGES, STAGE_BYTES, TRACE>(&tmA, &tmB, base, bars, num_kb, cid, ncl, rank, pairs_m, tiles_n,
                                              total_items, p);
  } else {
    setmaxnreg_inc<232>();
    const int ct = threadIdx.x - 128;               // consumer thread 0..255
    const int wg = ct >> 7, wi = (ct >> 5) & 3;
    const int fr = frag_row(wg, wi, lane);          // first of this thread's two fragment rows
    const int fc = 2 * (lane & 3);                  // column of this thread inside an 8-column block
    const uint32_t stage_u32 = base + STAGES * STAGE_BYTES;
    const bool issuer = ct == 0;
    RingPos<STAGES> pos;
    int cc = 0;
    float acc[BN / 2];
    [[maybe_unused]] float aff_rowsum[2] = {0.f, 0.f};   // affinity: row sums of this thread's two column slices
    [[maybe_unused]] float aff_mx = 1.f, aff_rmx = 1.f, aff_unscale = 1.f;
    [[maybe_unused]] unsigned long long* trec = nullptr;   // traced: this group's record of the current tile
    if constexpr (TRACE) trec = p.trace + blockIdx.x * trace_stride(total_items, ncl) + 4 + 4 * wg * ((total_items + ncl - 1) / ncl);
    const bool tracer = TRACE && (ct & 127) == 0;
    const NamedBar<1, EPI_THREADS> epi_bar;
    [[maybe_unused]] int mw = BN;   // affinity: columns of the tile this group's wgmmas compute (0: none)
    // each group computes 64 rows of the tile against the whole B slab
    auto mma = [&](int s, int kb) {
      const uint32_t sa = base + s * STAGE_BYTES;
      const uint64_t adesc = wgmma_desc_sw128(sa + wg * 64 * 128), bdesc = wgmma_desc_sw128(sa + A_ATOM_BYTES);
      if constexpr (EPI == EPI_AFFINITY_F32) mma_slab_cols(acc, mw, adesc, bdesc, kb == 0);
      else mma_slab<BN>(acc, adesc, bdesc, kb == 0);
    };
    // the slab was only read by wgmmas that have retired (wgmma_wait): nothing to publish, no release fence
    auto release = [&](int s) {
      if ((ct & 127) == 0) {
        mbar_arrive_cluster_relaxed(bars.empty(s), 0);
        mbar_arrive_cluster_relaxed(bars.empty(s), 1);
      }
    };
    for (int t = cid; t < total_items; t += ncl) {
      const TileCoord tc = decode_tile<BN>(t, pairs_m, tiles_n, rank, p.tri);
      if constexpr (EPI == EPI_AFFINITY_F32) {
        // No wgmma for what no output reads; the group still waits for and releases every slab, so the ring and the
        // pair's multicast run exactly as for a computed tile. The odd CTA's tile below the diagonal is discarded, a
        // group whose 64 rows all lie past the image computes nothing, and the image's last column tile runs on the
        // narrowest wgmma that covers its columns: the epilogue zeroes every column >= M and masks every row >= M,
        // so the stale accumulators past them reach no output.
        mw = (p.tri && tc.m0 > tc.n0) || tc.m0 + 64 * wg >= M ? 0 : mma_cols(min(N - tc.n0, BN));
      }
      if (tracer) trec[0] = globaltimer();
      const int last = consume_slabs(pos, bars, num_kb, tracer ? trec + 1 : nullptr, mma, release);
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (tracer) trec[2] = globaltimer();
      release(last);

      if constexpr (epi_uses_tma_store(EPI)) {
        // ---- 128-byte-wide output boxes (32 fp32 or 64 fp16 columns): fragments -> +bias (-> GELU) -> 128 B-swizzled
        // staging box -> one TMA store. The residual epilogue uses the TMA *reduce-add* (performed at the L2):
        // x += acc + bias never reads x.
        constexpr bool OUT16 = (EPI == DSS_EPI_BIAS_F16 || EPI == DSS_EPI_BIAS_GELU_F16);
        constexpr int BOXC = OUT16 ? 64 : 32;          // columns per 128-byte-wide store box
        constexpr int NBOX = BN / BOXC;
        if constexpr (EPI == EPI_AFFINITY_F32) {
          // the odd CTA's tile below the diagonal (its slabs only waited for and released, in step with the pair)
          if (p.tri && tc.m0 > tc.n0) {
            if (tracer) {   // no epilogue
              trec[3] = trec[2];
              trec += 4;
            }
            continue;
          }
        }
#pragma unroll
        for (int b = 0; b < NBOX; ++b) {
          const int nc = tc.n0 + b * BOXC;           // first global column of the box
          const bool live = nc < N;
          box_acquire(epi_bar, issuer);
          const uint32_t sbuf = stage_u32 + (cc & 1) * BOX_BYTES;
          if constexpr (EPI != EPI_AFFINITY_F32) {
#pragma unroll
            for (int i = 0; i < BOXC / 8; ++i) {
              const int ci = b * (BOXC / 8) + i;       // 8-column block of the tile
              const int col = nc + 8 * i + fc;         // global column of this thread's pair
              float2 bv = make_float2(0.f, 0.f);
              if (p.bias != nullptr && col < N) bv = __ldg(reinterpret_cast<const float2*>(p.bias + col));
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float x0 = acc[4 * ci + 2 * h] + bv.x, x1 = acc[4 * ci + 2 * h + 1] + bv.y;
                if constexpr (EPI == DSS_EPI_BIAS_GELU_F16) { x0 = gelu_erf(x0); x1 = gelu_erf(x1); }
                box_put_pair<OUT16>(sbuf, fr + 8 * h, i, lane, x0, x1);
              }
            }
          } else {
            // ---- affinity: the box (32 fp32 columns) goes through a row-major copy so that each thread can own one row
            // x 8 columns ("slice") as the degree fusion below needs: thread (quarter q = rows 32q.., slice pair sp)
            // handles slices 2 sp and 2 sp + 1
            float* rowbuf = stage_base + 2 * (BOX_BYTES / 4);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int ci = b * 4 + i;
#pragma unroll
              for (int h = 0; h < 2; ++h)
                *reinterpret_cast<float2*>(rowbuf + (fr + 8 * h) * STG_LD + 8 * i + fc) =
                    make_float2(acc[4 * ci + 2 * h], acc[4 * ci + 2 * h + 1]);
            }
            epi_bar.sync();
            const int q = (ct >> 5) & 3, sp = ct >> 7;
            const int row = q * 32 + lane;
            const int m = tc.m0 + row;
            if (b == 0) {   // per-tile constants (L2 round trips: not once per box)
              aff_mx = __uint_as_float(__ldg(p.img_max + tc.z));
              aff_rmx = __frcp_rn(aff_mx);
              // un-normalised features were pre-scaled by pre = 2^-ceil(log2 max|f|) (affinity.cu): the scale cancels
              // in W / max(W); when the division is skipped (which_matrix = 'affinity' / 'affinity_svd') it is undone
              aff_unscale = 1.0f;
              if ((p.threshold & 2) && p.img_absmax != nullptr) {
                const float am = __uint_as_float(__ldg(p.img_absmax + tc.z));
                if (am > 0.f) aff_unscale = exp2f(2.0f * ceilf(log2f(am)));
              }
              aff_rowsum[0] = aff_rowsum[1] = 0.f;
            }
            const bool upper = tc.m0 < tc.n0;
            // edge boxes only (last tile row / column of the image): the colour term and the bounds are per element
            const bool edge = nc + BOXC > M || tc.m0 + BM > M;   // (uniform)
            const bool rowok = !edge || m < M;
            float* part = p.deg_part + (long long)tc.z * (8 * tiles_n) * p.ld_part;
            float* Wz = reinterpret_cast<float*>(p.out) + (long long)tc.z * M * p.ldo;
#pragma unroll
            for (int hs = 0; hs < 2; ++hs) {
              constexpr int W = 8;
              const int sl = 2 * sp + hs;
              const int n = nc + sl * W;
              float x[W];
              {
                const float4 v0 = *reinterpret_cast<const float4*>(rowbuf + row * STG_LD + sl * W);
                const float4 v1 = *reinterpret_cast<const float4*>(rowbuf + row * STG_LD + sl * W + 4);
                x[0] = v0.x; x[1] = v0.y; x[2] = v0.z; x[3] = v0.w; x[4] = v1.x; x[5] = v1.y; x[6] = v1.z; x[7] = v1.w;
              }
              // W[z, m, n] = relu(acc) / max (+ lambda * counts); columns >= M (row-pitch padding) are zeros; rows >= M
              // are clipped by the per-image (3D) tensor map
              const float mx = aff_mx, rmx = aff_rmx, unscale = aff_unscale;
              const bool relu = p.threshold & 1, nodiv = p.threshold & 2;
              // y / mx without the compiler's IEEE division subroutine: its range check sends zero and tiny numerators
              // -- most of a thresholded affinity -- down a long slow path. mx is the largest Gram diagonal: exactly 1 for
              // most normalised images (nothing to do), else q = y r, one residual correction: q + (y - q mx) r -- the
              // correctly rounded quotient for these operand ranges (0 <= y <= ~mx, mx in the normal range).
              const bool scale = !nodiv && mx != 1.0f;
#pragma unroll
              for (int e = 0; e < W; ++e) {
                float y = x[e];
                if (relu) y = fmaxf(y, 0.f);                  // W * (W > 0)
                if (scale) {                                  // W / W.max()
                  const float q0 = y * rmx;
                  y = fmaf(fmaf(-q0, mx, y), rmx, q0);
                }
                if (nodiv) y *= unscale;
                x[e] = y;
              }
              if (p.counts != nullptr && rowok) {
                const uint8_t* cnt = p.counts + ((long long)tc.z * M + m) * M + n;
#pragma unroll
                for (int e = 0; e < W; ++e)
                  if (!edge || n + e < M) x[e] += static_cast<float>(cnt[e]) * p.lambda;   // + W_color * lambda
              }
              if (edge) {
#pragma unroll
                for (int e = 0; e < W; ++e)
                  if (n + e >= M) x[e] = 0.f;
              }
              if (p.tri) {
                // ---- symmetric mode. The matrix is exactly symmetric by construction (the same value is written to
                // (m, n) and (n, m)), only tiles on or above the diagonal do any work, and the degree D = W 1 that the
                // eigensolver starts from (extract_utils.py:207-220) is accumulated here instead of by another pass
                // over W: per-thread row sums and per-warp column sums go to fixed partial slots (deterministic order).
                // Tiles strictly above the diagonal: TMA store of the tile + mirrored direct stores. Diagonal tiles: the
                // two halves of the tile come out of differently ordered accumulations (the split-fp16 K groups are
                // swapped between the operands), so only the elements on or above the diagonal are stored -- each to
                // both positions -- and the TMA store is skipped: W[i, j] and W[j, i] are the same bits everywhere.
                float xm[W];
#pragma unroll
                for (int e = 0; e < W; ++e) {
                  xm[e] = rowok ? x[e] : 0.f;
                  aff_rowsum[hs] += xm[e];
                }
                if (b == NBOX - 1 && rowok)   // row partial slot of (column tile j, slice sl)
                  part[(long long)((tc.n0 / BN) * 4 + sl) * p.ld_part + m] = aff_rowsum[hs];
                if (!upper) {                 // diagonal tile: direct stores only, no staging / TMA store for this box
                  if (rowok) {
                    float* rowp = Wz + (long long)m * p.ldo + n;      // (m, n + e)
                    float* colp = Wz + (long long)n * p.ldo + m;      // (n + e, m)
#pragma unroll
                    for (int e = 0; e < W; ++e) {
                      if (n + e >= m && n + e < p.ldo) rowp[e] = x[e];                          // on / above the diagonal
                      if (n + e > m && n + e < M) colp[(long long)e * p.ldo] = x[e];            // its mirror image
                    }
                  }
                  continue;
                }
                // mirrored store W[z, n + e, m] = W[z, m, n + e]: lanes hold consecutive m -> 128 B per warp store
                if (!edge || m < p.ldo) {
                  float* colp = Wz + (long long)n * p.ldo + m;
#pragma unroll
                  for (int e = 0; e < W; ++e)
                    if (!edge || n + e < M) colp[(long long)e * p.ldo] = xm[e];
                }
                // column sums over this warp's 32 rows: segmented butterfly (8 -> 4 -> 2 -> 1 values per lane)
                float c4[4], c2[2], c1;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const float mine = (lane & 16) ? xm[e + 4] : xm[e], theirs = (lane & 16) ? xm[e] : xm[e + 4];
                  c4[e] = mine + __shfl_xor_sync(0xffffffffu, theirs, 16);
                }
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const float mine = (lane & 8) ? c4[e + 2] : c4[e], theirs = (lane & 8) ? c4[e] : c4[e + 2];
                  c2[e] = mine + __shfl_xor_sync(0xffffffffu, theirs, 8);
                }
                {
                  const float mine = (lane & 4) ? c2[1] : c2[0], theirs = (lane & 4) ? c2[0] : c2[1];
                  c1 = mine + __shfl_xor_sync(0xffffffffu, theirs, 4);
                }
                c1 += __shfl_xor_sync(0xffffffffu, c1, 2);
                c1 += __shfl_xor_sync(0xffffffffu, c1, 1);
                // lane l now holds the sum of column e = 4 * bit4 + 2 * bit3 + bit2 of l (all four lanes l & 3 agree)
                if ((lane & 3) == 0) {
                  const int e = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
                  // column partial slot of (row tile i = m0 / BM, lane quarter q); it belongs to matrix row n + e
                  part[(long long)(4 * tiles_n + (tc.m0 / BM) * 4 + q) * p.ld_part + n + e] = c1;
                }
              }
#pragma unroll
              for (int h = 0; h < 2; ++h) {   // two 16-byte chunks per slice
                const int j = sl * 2 + h;
                asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(sw128_addr(sbuf, row, j)),
                             "f"(x[h * 4 + 0]), "f"(x[h * 4 + 1]), "f"(x[h * 4 + 2]), "f"(x[h * 4 + 3])
                             : "memory");
              }
            }
            // diagonal tiles of the symmetric mode store directly (above) and skip the staging box
            if (p.tri && !upper) {
              epi_bar.sync();   // row-major copy reused by the next box
              continue;
            }
          }
          box_issue(epi_bar, issuer, [&, tc] {
            if (live) {
              if constexpr (EPI == DSS_EPI_BIAS_RESID_F32)
                tma_reduce_add_2d(&tmC, sbuf, nc, tc.m0);
              else if constexpr (EPI == EPI_AFFINITY_F32)
                tma_store_3d(&tmC, sbuf, nc, tc.m0, tc.z);
              else
                tma_store_2d(&tmC, sbuf, nc, tc.m0);
            }
          });
          ++cc;   // (boxes that skip the staging buffers -- diagonal affinity tiles -- do not advance the buffer parity)
        }
        if (tracer) {
          trec[3] = globaltimer();
          trec += 4;
        }
      } else {
        // ---- row-remapping epilogues: 32-column chunks through a row-major fp32 staging buffer (double buffered),
        // then row-contiguous (coalesced) global reads of the aux rows and writes of the result
#pragma unroll
        for (int c = 0; c < BN / 32; ++c, ++cc) {
          float* stg = stage_base + (cc & 1) * (STG_BYTES / 4);
          const int nc = tc.n0 + c * 32;           // global column of the chunk
          // Phase 1: +bias -> staging chunk (pitch 36 floats)
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int ci = c * 4 + i;
            float2 bv = make_float2(0.f, 0.f);
            if (p.bias != nullptr && nc < N) bv = __ldg(reinterpret_cast<const float2*>(p.bias + nc + 8 * i + fc));
#pragma unroll
            for (int h = 0; h < 2; ++h)
              *reinterpret_cast<float2*>(stg + (fr + 8 * h) * STG_LD + 8 * i + fc) =
                  make_float2(acc[4 * ci + 2 * h] + bv.x, acc[4 * ci + 2 * h + 1] + bv.y);
          }
          // Double-buffered staging: one barrier per chunk is enough, because a thread reaches the barrier of chunk c
          // only after finishing phase 2 of the previous user of buffer c^1.
          epi_bar.sync();
          // Phase 2: 8 lanes x 16 B cover the 128 B of one row of the chunk, 4 rows per warp instruction
          if (nc < N) {
            const int cw = ct >> 5;
            const int cl = (lane & 7) * 4;
            float4 v[4], y[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int rr = cw * 16 + i * 4 + (lane >> 3);
              const int m = tc.m0 + rr;
              v[i] = *reinterpret_cast<const float4*>(stg + rr * STG_LD + cl);
              y[i] = make_float4(0.f, 0.f, 0.f, 0.f);
              if (m < M) {
                if constexpr (EPI == DSS_EPI_PATCH_F32)
                  y[i] = __ldg(reinterpret_cast<const float4*>(p.aux + (long long)((m % p.rin) + 1) * p.ldo + nc + cl));
                if constexpr (EPI == EPI_PATCH_ROWS_F32)
                  y[i] = __ldg(reinterpret_cast<const float4*>(p.aux + out_row<EPI>(m, p) * p.ldo + nc + cl));
              }
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int rr = cw * 16 + i * 4 + (lane >> 3);
              const int m = tc.m0 + rr;
              if (m >= M) continue;
              float4 x = v[i];
              x.x += y[i].x; x.y += y[i].y; x.z += y[i].z; x.w += y[i].w;
              store_row4<EPI>(x, m, nc + cl, p);
            }
          }
        }
      }
    }
    if constexpr (epi_uses_tma_store(EPI)) {
      if (issuer) tma_store_wait_all<0>();
    }
  }
  cluster_pair_exit();
}

// ---------------------------------------------------------------------------------------------------------------
// Ping-pong schedule for the TMA-store epilogues. Item i of the CTA (t = cid + i * ncl, the same sequence in both CTAs
// of the pair) belongs to consumer group i % 2, so the ring holds the groups' slabs alternately, num_kb at a time, and
// a slot is released by one group in each CTA. Named barriers (IDs 1 + g: group g may issue; 3 + g: group g's
// epilogue) order the groups: item i > 0 waits (bar.sync, 256 threads) until the group of item i - 1 has issued its
// last wgmma and arrived (bar.arrive) -- which that group does only when an item i exists, so every arrive has exactly
// one matching sync, for any number of items per CTA (an idle group waits for nothing and is waited for by nothing).
// The turn also keeps the parity waits on the full barriers sound: when a group starts item i, every slab of the items
// before it has arrived, so the previous use of each slot it waits on has completed (a wait is never two phases ahead).
// Each output element sums the same K slabs in the same order as under the cooperative schedule.
constexpr int PP_TURN_BAR = 1, PP_EPI_BAR = 3;
template <int EPI, bool TRACE = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_f16_pingpong_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                         const __grid_constant__ CUtensorMap tmC, int M, int N, int K, int pairs_m, int tiles_n,
                         int total_items, EpiParams p) {
  static_assert(epi_uses_tma_store(EPI) && EPI != EPI_AFFINITY_F32, "ping-pong: the four ViT epilogues only");
  constexpr int BN = PP_BN;
  using Cfg = TileCfg<EPI, BN, true>;
  constexpr int STAGES = Cfg::STAGES, STAGE_BYTES = Cfg::STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;   // SWIZZLE_128B alignment
  const RingBars<STAGES> bars{base + STAGES * STAGE_BYTES + Cfg::STAGING_BYTES};

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_kb = (K + BK - 1) / BK;
  const int rank = (int)cluster_ctarank();
  const int cid = blockIdx.x >> 1, ncl = gridDim.x >> 1;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmC);
    bars.init(2);   // one consumer group of each CTA
    mbar_fence_init();
  }
  __syncthreads();
  cluster_sync_all();

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0)
      produce<BN, STAGES, STAGE_BYTES, TRACE>(&tmA, &tmB, base, bars, num_kb, cid, ncl, rank, pairs_m, tiles_n,
                                              total_items, p);
  } else {
    setmaxnreg_inc<232>();
    const int ct = threadIdx.x - 128;
    const int wg = ct >> 7, wi = (ct >> 5) & 3;
    const int fc = 2 * (lane & 3);
    const bool issuer = (ct & 127) == 0;   // issues this group's stores and releases its slabs
    const uint32_t stage_u32 = base + STAGES * STAGE_BYTES + wg * 2 * BOX_BYTES;   // this group's two boxes
    RingPos<STAGES> pos;
    int cc = 0;
    if (wg == 1) pos.skip(num_kb);   // the ring position of item 1: item 0's slabs come first
    float acc[2][64];   // rows 0-63 and 64-127 of the tile
    [[maybe_unused]] unsigned long long* trec = nullptr;
    if constexpr (TRACE) trec = p.trace + blockIdx.x * trace_stride(total_items, ncl) + 4 + 4 * wg * ((total_items + ncl - 1) / ncl);
    const bool tracer = TRACE && issuer;
    const GroupBar<128> epi_bar{PP_EPI_BAR + wg};
    auto mma = [&](int s, int kb) {
      const uint32_t sa = base + s * STAGE_BYTES;
      mma_slab<BN, 2>(acc, {wgmma_desc_sw128(sa), wgmma_desc_sw128(sa + 64 * 128)}, wgmma_desc_sw128(sa + A_ATOM_BYTES),
                      kb == 0);
    };
    auto release = [&](int s) {
      if ((ct & 127) == 0) {
        mbar_arrive_cluster_relaxed(bars.empty(s), 0);
        mbar_arrive_cluster_relaxed(bars.empty(s), 1);
      }
    };
    for (int t = cid + wg * ncl; t < total_items; t += 2 * ncl) {
      if (t != cid) {   // wait for the MMA turn
        __syncwarp();
        asm volatile("bar.sync %0, 256;" ::"r"(PP_TURN_BAR + wg) : "memory");
      }
      const TileCoord tc = decode_tile<BN>(t, pairs_m, tiles_n, rank);
      if (tracer) trec[0] = globaltimer();
      const int last = consume_slabs(pos, bars, num_kb, tracer ? trec + 1 : nullptr, mma, release);
      // hand the MMA turn to the group of the next item (its wgmmas queue behind this tile's last ones)
      if (t + ncl < total_items) {
        __syncwarp();
        asm volatile("bar.arrive %0, 256;" ::"r"(PP_TURN_BAR + (wg ^ 1)) : "memory");
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc[0]);
      wgmma_fence_acc(acc[1]);
      if (tracer) trec[2] = globaltimer();
      release(last);
      pos.skip(num_kb);   // the other group's item

      // ---- epilogue, as in the cooperative kernel but on this group's 128 rows and boxes: +bias (-> GELU) -> 128 B-
      // swizzled staging box -> TMA store / reduce-add
      constexpr bool OUT16 = (EPI == DSS_EPI_BIAS_F16 || EPI == DSS_EPI_BIAS_GELU_F16);
      constexpr int BOXC = OUT16 ? 64 : 32;
      constexpr int NBOX = BN / BOXC;
#pragma unroll
      for (int b = 0; b < NBOX; ++b) {
        const int nc = tc.n0 + b * BOXC;
        box_acquire(epi_bar, issuer);
        const uint32_t sbuf = stage_u32 + (cc & 1) * BOX_BYTES;
#pragma unroll
        for (int i = 0; i < BOXC / 8; ++i) {
          const int ci = b * (BOXC / 8) + i;
          const int col = nc + 8 * i + fc;
          float2 bv = make_float2(0.f, 0.f);
          if (p.bias != nullptr && col < N) bv = __ldg(reinterpret_cast<const float2*>(p.bias + col));
#pragma unroll
          for (int hr = 0; hr < 4; ++hr) {   // row half hr / 2, fragment row + 8 (hr % 2)
            const int h = hr >> 1, e = hr & 1;
            const int row = frag_row(h, wi, lane) + 8 * e;
            float x0 = acc[h][4 * ci + 2 * e] + bv.x, x1 = acc[h][4 * ci + 2 * e + 1] + bv.y;
            // the next tile's first wgmma ignores the accumulators (scale-d 0), but its asm reads them: constants
            // instead of values let the registers serve the rest of this epilogue
            acc[h][4 * ci + 2 * e] = acc[h][4 * ci + 2 * e + 1] = 0.f;
            if constexpr (EPI == DSS_EPI_BIAS_GELU_F16) { x0 = gelu_erf(x0); x1 = gelu_erf(x1); }
            box_put_pair<OUT16>(sbuf, row, i, lane, x0, x1);
          }
        }
        box_issue(epi_bar, issuer, [&] {
          if (nc < N) {
            if constexpr (EPI == DSS_EPI_BIAS_RESID_F32)
              tma_reduce_add_2d(&tmC, sbuf, nc, tc.m0);
            else
              tma_store_2d(&tmC, sbuf, nc, tc.m0);
          }
        });
        ++cc;
      }
      if (tracer) {
        trec[3] = globaltimer();
        trec += 4;
      }
    }
    if (issuer) tma_store_wait_all<0>();
  }
  cluster_pair_exit();
}

// ---------------------------------------------------------------------------------------------------------------
// CUDA-core checker with the same epilogues (tests only).
template <int EPI>
__global__ void gemm_f16_simt_kernel(const __half* __restrict__ A, const __half* __restrict__ Wt, int M, int N, int K,
                                     EpiParams p) {
  // one thread = one row x 32 columns
  const int m = blockIdx.y * blockDim.y + threadIdx.y;
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) * 32;
  if (m >= M || n >= N) return;
  float v[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = 0.f;
  for (int k = 0; k < K; ++k) {
    const float a = __half2float(A[(size_t)m * K + k]);
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = fmaf(a, __half2float(Wt[(size_t)(n + j) * K + k]), v[j]);
  }
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] += p.bias[n + j];
  epilogue_store<EPI>(v, m, n, p);
}

// ---------------------------------------------------------------------------------------------------------------
// Host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess || !ptr) {
    set_error("cuTensorMapEncodeTiled not available from the CUDA driver");
    return nullptr;
  }
  fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  return fn;
}

// Tiled tensor map of `rank` dimensions (innermost first) with the settings all of them share: dense, 128 B swizzle,
// 256 B L2 promotion, zero fill out of bounds. `what` names the map in the error message; a 2D map's message also
// gives its rows and columns.
static int encode_tmap(CUtensorMap* tm, CUtensorMapDataType dtype, cuuint32_t rank, const void* ptr,
                       const cuuint64_t* gdim, const cuuint64_t* gstride, const cuuint32_t* box, const char* what) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return DSS_ERR_CUDA;
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, dtype, rank, const_cast<void*>(ptr), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    if (rank == 2)
      set_error("cuTensorMapEncodeTiled%s failed with CUresult %d (rows=%d cols=%d)", what, (int)r, (int)gdim[1],
                (int)gdim[0]);
    else
      set_error("cuTensorMapEncodeTiled%s failed with CUresult %d", what, (int)r);
    return DSS_ERR_CUDA;
  }
  return DSS_OK;
}

// Tile width the weight tensor maps of the TMA-store epilogues (the ping-pong schedule) are built for.
int gemm_tile_n() { return PP_BN; }

// Tile width of the cooperative schedule for an N-column GEMM: the widest of 256 / 192 / 128 that divides N (operand
// bytes per FLOP fall with BN).
static int coop_tile_n(int N) { return N % 256 == 0 ? 256 : (N % 192 == 0 ? 192 : 128); }

// 2D fp16 row-major [rows, cols] tensor, box = 64 columns x box_rows rows, 128 B swizzle, zero fill out of bounds.
int make_tmap_f16(CUtensorMap* tm, const void* ptr, int rows, int cols, int box_rows) {
  if (!get_encode_fn()) return DSS_ERR_CUDA;
  DSS_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA operand must be 16-byte aligned");
  DSS_REQUIRE(cols % 8 == 0, "TMA operand row pitch must be a multiple of 16 bytes (cols=%d)", cols);
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * 2};
  DSS_REQUIRE(box_rows > 0 && box_rows <= 256, "TMA box rows must be in [1, 256]");
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  return encode_tmap(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, ptr, gdim, gstride, box, "");
}

// Output tensor map for the TMA-store epilogues: row-major [rows, cols] of fp16 (box 64 x 128) or fp32 (box 32 x 128),
// i.e. 128-byte-wide boxes with the 128 B swizzle.
int make_tmap_out(CUtensorMap* tm, const void* ptr, int rows, int cols, int is_f32) {
  if (!get_encode_fn()) return DSS_ERR_CUDA;
  DSS_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA output must be 16-byte aligned");
  const int esz = is_f32 ? 4 : 2;
  DSS_REQUIRE((cols * esz) % 16 == 0, "TMA output row pitch must be a multiple of 16 bytes (cols=%d)", cols);
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * esz};
  cuuint32_t box[2] = {(cuuint32_t)(is_f32 ? 32 : 64), (cuuint32_t)BM};
  return encode_tmap(tm, is_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, ptr, gdim,
                     gstride, box, " (output)");
}

// Per-image fp32 output [images, rows, ld] for the affinity epilogue: 3D map, box 32 columns x 128 rows x 1 image
int make_tmap_out3d_f32(CUtensorMap* tm, const void* ptr, int images, int rows, int ld) {
  if (!get_encode_fn()) return DSS_ERR_CUDA;
  DSS_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && ld % 4 == 0, "affinity output must be 16-byte aligned / pitched");
  cuuint64_t gdim[3] = {(cuuint64_t)ld, (cuuint64_t)rows, (cuuint64_t)images};
  cuuint64_t gstride[2] = {(cuuint64_t)ld * 4, (cuuint64_t)rows * ld * 4};
  cuuint32_t box[3] = {32, (cuuint32_t)BM, 1};
  return encode_tmap(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, ptr, gdim, gstride, box, " (3D output)");
}

// 3D fp16 output [images, rows, cols] written in 128-row x 64-column boxes (128 B swizzle); rows past `rows` of an image
// are clipped by the TMA unit, so a partial last tile never spills into the next image.
int make_tmap_out3d_f16(CUtensorMap* tm, const void* ptr, int images, int rows, int cols) {
  if (!get_encode_fn()) return DSS_ERR_CUDA;
  DSS_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && cols % 64 == 0, "fp16 tile output must be 16-byte aligned, cols %% 64 == 0");
  cuuint64_t gdim[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)images};
  cuuint64_t gstride[2] = {(cuuint64_t)cols * 2, (cuuint64_t)rows * cols * 2};
  cuuint32_t box[3] = {64, (cuuint32_t)BM, 1};
  return encode_tmap(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, ptr, gdim, gstride, box, " (3D fp16 output)");
}

// PP: ping-pong schedule (BN == PP_BN), else cooperative; TRACE: the phase-traced instantiation (p.trace)
template <int EPI, int BN, bool PP = false, bool TRACE = false>
static int launch_tc_bn(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap* tmC, int M, int N, int K,
                        const EpiParams& p, cudaStream_t st, int kclass, int batch) {
  static_assert(!PP || BN == PP_BN, "ping-pong tile width");
  constexpr auto kernel = [] {
    if constexpr (PP) return gemm_f16_pingpong_kernel<EPI, TRACE>;
    else return gemm_f16_wgmma_kernel<EPI, BN, TRACE>;
  }();
  const int pairs_m = cdiv(cdiv(M, BM), 2), tiles_n = cdiv(N, BN);
  int per_img = pairs_m * tiles_n;
  if (p.tri) {   // symmetric output: row pair p visits the n-tiles j >= 2p only (see decode_tile)
    per_img = 0;
    for (int q = 0; q < pairs_m; ++q) per_img += tiles_n - 2 * q > 0 ? tiles_n - 2 * q : 0;
  }
  const int total = per_img * batch;   // work items of a CTA pair
  if (epi_uses_tma_store(EPI) && tmC == nullptr) {
    set_error("gemm: this epilogue needs an output tensor map");
    return DSS_ERR_BAD_ARG;
  }
  return launch_cluster_pairs<kernel, TileCfg<EPI, BN, PP>::SMEM_BYTES>(gemm_clusters(total), GEMM_THREADS, st, kclass,
                                                                        tmA, tmB, tmC ? *tmC : tmA, M, N, K, pairs_m,
                                                                        tiles_n, total, p);
}

// Cooperative schedule; bn = tile width the B tensor map was built for (its TMA box has bn / 2 rows)
template <int EPI, bool TRACE = false>
static int launch_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap* tmC, int M, int N, int K,
                     const EpiParams& p, cudaStream_t st, int kclass, int bn, int batch = 1) {
  switch (bn) {
    case 128: return launch_tc_bn<EPI, 128, false, TRACE>(tmA, tmB, tmC, M, N, K, p, st, kclass, batch);
    case 192:
      if constexpr (epi_uses_tma_store(EPI) && EPI != EPI_AFFINITY_F32)
        return launch_tc_bn<EPI, 192, false, TRACE>(tmA, tmB, tmC, M, N, K, p, st, kclass, batch);
      break;
    case 256:
      if constexpr (epi_uses_tma_store(EPI) && EPI != EPI_AFFINITY_F32)
        return launch_tc_bn<EPI, 256, false, TRACE>(tmA, tmB, tmC, M, N, K, p, st, kclass, batch);
      break;
  }
  set_error("gemm: unsupported tile width %d", bn);
  return DSS_ERR_BAD_ARG;
}

// Ping-pong schedule (the B tensor map's box has PP_BN / 2 rows)
template <int EPI, bool TRACE = false>
static int launch_pp(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap* tmC, int M, int N, int K,
                     const EpiParams& p, cudaStream_t st, int kclass, int bn) {
  if (bn != PP_BN) {
    set_error("gemm: the weight tensor map must be built for tile width %d (got %d)", PP_BN, bn);
    return DSS_ERR_BAD_ARG;
  }
  return launch_tc_bn<EPI, PP_BN, true, TRACE>(tmA, tmB, tmC, M, N, K, p, st, kclass, 1);
}

static int check_gemm_args(int M, int N, int K, int epi, const float* bias, const void* out, const float* aux,
                           int rin, int rout) {
  DSS_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
  DSS_REQUIRE(N % 32 == 0 && K % 8 == 0, "gemm: need N %% 32 == 0 and K %% 8 == 0 (N=%d K=%d)", N, K);
  DSS_REQUIRE(bias && out, "gemm: null bias/out");
  if (epi == DSS_EPI_PATCH_F32 || epi == DSS_EPI_DROPCLS_F32) {
    DSS_REQUIRE(rin > 0 && rout > 0 && M % rin == 0, "gemm: bad row remap rin=%d rout=%d M=%d", rin, rout, M);
    if (epi == DSS_EPI_PATCH_F32) DSS_REQUIRE(aux != nullptr, "gemm: patch epilogue needs aux (pos embed)");
  }
  return DSS_OK;
}

// Launch with pre-built tensor maps (used by the ViT forward, which caches them).
int gemm_f16_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap* tmC, const float* bias, void* out,
                int M, int N, int K, int epi, const float* aux, int rin, int rout, cudaStream_t st, int kclass, int bn) {
  int rc = check_gemm_args(M, N, K, epi, bias, out, aux, rin, rout);
  if (rc) return rc;
  EpiParams p{out, bias, aux, N, rin, rout, 0, nullptr, nullptr, nullptr, 0.f, 0, 0, 0, nullptr, 0};
  switch (epi) {
    case DSS_EPI_BIAS_F16: return launch_pp<DSS_EPI_BIAS_F16>(tmA, tmB, tmC, M, N, K, p, st, kclass, bn);
    case DSS_EPI_BIAS_GELU_F16: return launch_pp<DSS_EPI_BIAS_GELU_F16>(tmA, tmB, tmC, M, N, K, p, st, kclass, bn);
    case DSS_EPI_BIAS_RESID_F32: return launch_pp<DSS_EPI_BIAS_RESID_F32>(tmA, tmB, tmC, M, N, K, p, st, kclass, bn);
    case DSS_EPI_BIAS_F32: return launch_pp<DSS_EPI_BIAS_F32>(tmA, tmB, tmC, M, N, K, p, st, kclass, bn);
    case DSS_EPI_PATCH_F32: return launch_tc<DSS_EPI_PATCH_F32>(tmA, tmB, tmC, M, N, K, p, st, kclass, bn);
    case DSS_EPI_DROPCLS_F32: return launch_tc<DSS_EPI_DROPCLS_F32>(tmA, tmB, tmC, M, N, K, p, st, kclass, bn);
  }
  set_error("gemm: unknown epilogue %d", epi);
  return DSS_ERR_BAD_ARG;
}

// The row-table forms of the patch and DROPCLS epilogues (ragged ViT batches): GEMM row m goes to output row
// row_map[m] (device, -1: skip); the patch epilogue adds positional row row_map[m] of aux. Cooperative schedule, bn 128.
int gemm_f16_tc_rows(const CUtensorMap& tmA, const CUtensorMap& tmB, const float* bias, void* out, int M, int N, int K,
                     int epi, const float* aux, const int* row_map, cudaStream_t st, int kclass) {
  int rc = check_gemm_args(M, N, K, DSS_EPI_BIAS_F32, bias, out, aux, 0, 0);
  if (rc) return rc;
  DSS_REQUIRE(row_map, "gemm: row-table epilogue needs row_map");
  EpiParams p{out, bias, aux, N, 0, 0, 0, nullptr, nullptr, nullptr, 0.f, 0, 0, 0, nullptr, 0, nullptr, row_map};
  if (epi == DSS_EPI_PATCH_F32) {
    DSS_REQUIRE(aux != nullptr, "gemm: patch epilogue needs aux (pos embed)");
    return launch_tc<EPI_PATCH_ROWS_F32>(tmA, tmB, nullptr, M, N, K, p, st, kclass, 128);
  }
  if (epi == DSS_EPI_DROPCLS_F32) return launch_tc<EPI_DROPCLS_ROWS_F32>(tmA, tmB, nullptr, M, N, K, p, st, kclass, 128);
  set_error("gemm: no row-table form of epilogue %d", epi);
  return DSS_ERR_BAD_ARG;
}

// Batched Gram product for the affinity build: per image z, W[z] = epilogue(S[z] S'[z]^T) with S = split-fp16 rows
// [images*Nimg, 3d] (see affinity.cu). The GEMM's ncols output columns (Nimg <= ncols <= ldw) are the first ncols of
// the row pitch ldw; they also set the column tiles, and with them the layout of the degree partial slots
// [images, 8 * cdiv(ncols, 128), ld_part] that degree_reduce_kernel reads back. With `trace` (dss_debug_affinity_trace)
// the phase-traced instantiation runs; trace_bytes must hold trace_stride(items, clusters) words per CTA.
int affinity_gemm_tc(const CUtensorMap& tmS, const CUtensorMap& tmS_half, int images, int Nimg, int d, float* Wout, int ldw,
                     int ncols, const unsigned int* img_max, const unsigned int* img_absmax, const uint8_t* counts,
                     float lambda, int threshold, float* deg_part, int ld_part, cudaStream_t st,
                     unsigned long long* trace, size_t trace_bytes) {
  EpiParams p{Wout, nullptr, nullptr, ldw, 0, 0, Nimg, img_max, img_absmax, counts, lambda, threshold, d / BK,
              1, deg_part, ld_part, trace};
  DSS_REQUIRE(d % BK == 0, "affinity: feature dim must be a multiple of %d for the tensor-core path (got %d)", BK, d);
  DSS_REQUIRE(ncols >= Nimg && ncols <= ldw, "affinity: bad GEMM column count %d (N=%d ldw=%d)", ncols, Nimg, ldw);
  DSS_REQUIRE(deg_part != nullptr && ld_part >= cdiv(ncols, 128) * 128, "affinity: bad degree partial buffer");
  CUtensorMap tmW;
  int rc = make_tmap_out3d_f32(&tmW, Wout, images, Nimg, ldw);
  if (rc) return rc;
  if (trace == nullptr)
    return launch_tc<EPI_AFFINITY_F32>(tmS, tmS_half, &tmW, Nimg, ncols, 3 * d, p, st, KC_AFFINITY, 128, images);
  const int tiles = cdiv(ncols, 128);
  int items = 0;
  for (int q = 0; q < cdiv(cdiv(Nimg, BM), 2); ++q) items += tiles - 2 * q > 0 ? tiles - 2 * q : 0;
  items *= images;
  const int clusters = gemm_clusters(items);
  const size_t need = (size_t)(2 * clusters) * trace_stride(items, clusters) * sizeof(unsigned long long);
  DSS_REQUIRE(trace_bytes >= need, "debug_affinity_trace: the trace needs %zu bytes", need);
  DSS_CHECK_CUDA(cudaMemsetAsync(trace, 0, need, st));
  return launch_tc<EPI_AFFINITY_F32, true>(tmS, tmS_half, &tmW, Nimg, ncols, 3 * d, p, st, KC_AFFINITY, 128, images);
}

template <int EPI>
static int launch_simt(const void* A, const void* Wt, int M, int N, int K, const EpiParams& p, cudaStream_t st) {
  dim3 block(4, 32);
  dim3 grid(cdiv(N / 32, 4), cdiv(M, 32));
  LaunchScope scope(st, KC_MISC);
  gemm_f16_simt_kernel<EPI><<<grid, block, 0, st>>>(reinterpret_cast<const __half*>(A),
                                                    reinterpret_cast<const __half*>(Wt), M, N, K, p);
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

}  // namespace dss

using namespace dss;

extern "C" int dss_op_gemm_f16(const void* A, const void* Wt, const float* bias, void* out, int M, int N, int K,
                               int epilogue, const float* aux, int rin, int rout, dss_stream_t stream) {
  int rc = check_gemm_args(M, N, K, epilogue, bias, out, aux, rin, rout);
  if (rc) return rc;
  DSS_REQUIRE(A && Wt, "gemm: null operand");
  CUtensorMap tmA, tmB;
  const int bn = epi_uses_tma_store(epilogue) ? gemm_tile_n() : 128;   // row-remapping epilogues: 128-wide only
  if ((rc = make_tmap_f16(&tmA, A, M, K, BM))) return rc;
  if ((rc = make_tmap_f16(&tmB, Wt, N, K, bn / 2))) return rc;   // each CTA of a pair loads (and multicasts) half a tile
  CUtensorMap tmC;
  const bool tma_out = epi_uses_tma_store(epilogue);
  if (tma_out) {
    const int f32 = (epilogue == DSS_EPI_BIAS_RESID_F32 || epilogue == DSS_EPI_BIAS_F32) ? 1 : 0;
    if ((rc = make_tmap_out(&tmC, out, M, N, f32))) return rc;
  }
  return gemm_f16_tc(tmA, tmB, tma_out ? &tmC : nullptr, bias, out, M, N, K, epilogue, aux, rin, rout,
                     static_cast<cudaStream_t>(stream), KC_GEMM_OTHER, bn);
}

extern "C" int dss_op_gemm_f16_simt(const void* A, const void* Wt, const float* bias, void* out, int M, int N, int K,
                                    int epilogue, const float* aux, int rin, int rout, dss_stream_t stream) {
  int rc = check_gemm_args(M, N, K, epilogue, bias, out, aux, rin, rout);
  if (rc) return rc;
  DSS_REQUIRE(A && Wt, "gemm: null operand");
  EpiParams p{out, bias, aux, N, rin, rout, 0, nullptr, nullptr, nullptr, 0.f, 0, 0, 0, nullptr, 0};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (epilogue) {
    case DSS_EPI_BIAS_F16: return launch_simt<DSS_EPI_BIAS_F16>(A, Wt, M, N, K, p, st);
    case DSS_EPI_BIAS_GELU_F16: return launch_simt<DSS_EPI_BIAS_GELU_F16>(A, Wt, M, N, K, p, st);
    case DSS_EPI_BIAS_RESID_F32: return launch_simt<DSS_EPI_BIAS_RESID_F32>(A, Wt, M, N, K, p, st);
    case DSS_EPI_BIAS_F32: return launch_simt<DSS_EPI_BIAS_F32>(A, Wt, M, N, K, p, st);
    case DSS_EPI_PATCH_F32: return launch_simt<DSS_EPI_PATCH_F32>(A, Wt, M, N, K, p, st);
    case DSS_EPI_DROPCLS_F32: return launch_simt<DSS_EPI_DROPCLS_F32>(A, Wt, M, N, K, p, st);
  }
  set_error("gemm: unknown epilogue %d", epilogue);
  return DSS_ERR_BAD_ARG;
}

// Tuning probe (not used by the product path): plain bias epilogue with an explicit tile width (`stages` is ignored).
extern "C" int dss_debug_gemm_cfg(const void* A, const void* Wt, const float* bias, void* out, int M, int N, int K,
                                  int bn, int stages, dss_stream_t stream) {
  int rc = check_gemm_args(M, N, K, DSS_EPI_BIAS_F16, bias, out, nullptr, 0, 0);
  if (rc) return rc;
  CUtensorMap tmA, tmB, tmC;
  if ((rc = make_tmap_f16(&tmA, A, M, K, BM))) return rc;
  if ((rc = make_tmap_f16(&tmB, Wt, N, K, bn / 2))) return rc;
  if ((rc = make_tmap_out(&tmC, out, M, N, 0))) return rc;
  EpiParams p{out, bias, nullptr, N, 0, 0, 0, nullptr, nullptr, nullptr, 0.f, 0, 0, 0, nullptr, 0};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  (void)stages;   // the ring depth follows from the shared-memory budget of the tile width
  switch (bn) {
    case 128: return launch_tc_bn<DSS_EPI_BIAS_F16, 128>(tmA, tmB, &tmC, M, N, K, p, st, KC_GEMM_OTHER, 1);
    case 192: return launch_tc_bn<DSS_EPI_BIAS_F16, 192>(tmA, tmB, &tmC, M, N, K, p, st, KC_GEMM_OTHER, 1);
    case 256: return launch_tc_bn<DSS_EPI_BIAS_F16, 256>(tmA, tmB, &tmC, M, N, K, p, st, KC_GEMM_OTHER, 1);
  }
  set_error("debug_gemm_cfg: unsupported (bn=%d, stages=%d)", bn, stages);
  return DSS_ERR_BAD_ARG;
}

namespace dss {
template <int EPI, bool TRACE>
static int launch_schedule(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, int M, int N, int K,
                           const EpiParams& p, cudaStream_t st, int schedule, int bn) {
  return schedule ? launch_pp<EPI, TRACE>(tmA, tmB, &tmC, M, N, K, p, st, KC_GEMM_OTHER, bn)
                  : launch_tc<EPI, TRACE>(tmA, tmB, &tmC, M, N, K, p, st, KC_GEMM_OTHER, bn);
}

// One of the four TMA-store epilogues under either schedule (0 = cooperative at coop_tile_n(N), 1 = ping-pong), traced
// when `trace` is not null (trace_bytes must hold trace_stride(items, clusters) words per CTA).
template <bool TRACE>
static int debug_gemm_schedule(const void* A, const void* Wt, const float* bias, void* out, int M, int N, int K,
                               int epilogue, int schedule, unsigned long long* trace, size_t trace_bytes,
                               cudaStream_t st) {
  int rc = check_gemm_args(M, N, K, epilogue, bias, out, nullptr, 0, 0);
  if (rc) return rc;
  DSS_REQUIRE(A && Wt, "gemm: null operand");
  DSS_REQUIRE(epi_uses_tma_store(epilogue), "debug_gemm_schedule: epilogue %d is not one of the four ViT epilogues", epilogue);
  DSS_REQUIRE(schedule == 0 || schedule == 1, "debug_gemm_schedule: schedule must be 0 (cooperative) or 1 (ping-pong)");
  const int bn = schedule ? PP_BN : coop_tile_n(N);
  if (TRACE) {
    const int items = cdiv(cdiv(M, BM), 2) * cdiv(N, bn), clusters = gemm_clusters(items);
    const size_t need = (size_t)(2 * clusters) * trace_stride(items, clusters) * sizeof(unsigned long long);
    DSS_REQUIRE(trace != nullptr && trace_bytes >= need, "debug_gemm_trace: the trace needs %zu bytes", need);
    DSS_CHECK_CUDA(cudaMemsetAsync(trace, 0, need, st));
  }
  CUtensorMap tmA, tmB, tmC;
  if ((rc = make_tmap_f16(&tmA, A, M, K, BM))) return rc;
  if ((rc = make_tmap_f16(&tmB, Wt, N, K, bn / 2))) return rc;
  const int f32 = (epilogue == DSS_EPI_BIAS_RESID_F32 || epilogue == DSS_EPI_BIAS_F32) ? 1 : 0;
  if ((rc = make_tmap_out(&tmC, out, M, N, f32))) return rc;
  EpiParams p{out, bias, nullptr, N, 0, 0, 0, nullptr, nullptr, nullptr, 0.f, 0, 0, 0, nullptr, 0, trace};
  switch (epilogue) {
    case DSS_EPI_BIAS_F16: return launch_schedule<DSS_EPI_BIAS_F16, TRACE>(tmA, tmB, tmC, M, N, K, p, st, schedule, bn);
    case DSS_EPI_BIAS_GELU_F16: return launch_schedule<DSS_EPI_BIAS_GELU_F16, TRACE>(tmA, tmB, tmC, M, N, K, p, st, schedule, bn);
    case DSS_EPI_BIAS_RESID_F32: return launch_schedule<DSS_EPI_BIAS_RESID_F32, TRACE>(tmA, tmB, tmC, M, N, K, p, st, schedule, bn);
    case DSS_EPI_BIAS_F32: return launch_schedule<DSS_EPI_BIAS_F32, TRACE>(tmA, tmB, tmC, M, N, K, p, st, schedule, bn);
  }
  set_error("debug_gemm_schedule: unknown epilogue %d", epilogue);
  return DSS_ERR_BAD_ARG;
}
}  // namespace dss

extern "C" int dss_debug_gemm_schedule(const void* A, const void* Wt, const float* bias, void* out, int M, int N, int K,
                                       int epilogue, int schedule, dss_stream_t stream) {
  return debug_gemm_schedule<false>(A, Wt, bias, out, M, N, K, epilogue, schedule, nullptr, 0,
                                    static_cast<cudaStream_t>(stream));
}

extern "C" int dss_debug_gemm_trace(const void* A, const void* Wt, const float* bias, void* out, int M, int N, int K,
                                    int epilogue, int schedule, unsigned long long* trace, size_t trace_bytes,
                                    dss_stream_t stream) {
  return debug_gemm_schedule<true>(A, Wt, bias, out, M, N, K, epilogue, schedule, trace, trace_bytes,
                                   static_cast<cudaStream_t>(stream));
}
