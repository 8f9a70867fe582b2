// LayerNorm fused into an A-stationary wgmma GEMM for the K = 384 layers of ViT-S (qkv and fc1):
//     out[M, N] (f16) = epilogue( LayerNorm(x[M, 384]; gamma, beta, eps) @ Wt[N, 384]^T + bias )
// The stand-alone LayerNorm kernel and the fp16 round trip of its output disappear: three warps of the CTA read the
// fp32 residual stream, normalise it and write the fp16 A operand straight into shared memory in the layout wgmma
// reads (K-major rows of 128 bytes, 128 B swizzle -- what a TMA box {64 x f16, 128 rows} would have written). The
// 128 x 384 panel (96 KB) then stays put while the weight tiles of ALL n-tiles stream past it through a TMA ring.
//
// One CTA per SM, CTAs in clusters of two that walk the same n-tiles for two vertically adjacent 128-row blocks; each
// CTA fetches half of every weight tile and multicasts it into both (as gemm.cu does).
//   warp 0            TMA producer of the weight ring
//   warps 1..3        LayerNorm producers: row statistics of the NEXT row block are computed while the current
//                     block's wgmmas run (x is read once from HBM; the second read below hits the L2); once the MMA
//                     groups have released the panel, the rows are re-read, normalised and written
//   warp groups 1, 2  wgmma m64 x BN x 16 on 64 rows each, epilogue from the register accumulators (+bias -> GELU ->
//                     fp16 -> swizzled staging box -> TMA store)
// The normalisation is layernorm_f16_kernel's arithmetic (the ln_* helpers of common.cuh, every rounding explicit), so
// the A operand is bit for bit the stand-alone kernel's output.
#include <math.h>

#include "gemm_pipeline.cuh"

namespace dss {

constexpr int LG_BM = 128, LG_K = 384, LG_SLABS = LG_K / BK, LG_SLAB_BYTES = LG_BM * 128;
constexpr int LG_THREADS = 384, LG_LN_WARPS = 3;
constexpr int LG_BOX_BYTES = LG_BM * 128;

template <int BN> struct LnCfg {
  static constexpr int A_BYTES = LG_SLABS * LG_SLAB_BYTES;          // 96 KB
  static constexpr int B_STAGE = BN * 128;                          // BN rows x 64 f16
  static constexpr int STAGING = 2 * LG_BOX_BYTES;
  static constexpr int VEC_BYTES = 2 * LG_BM * 4;                   // row sum[128], rstd[128]
  static constexpr int FIXED = A_BYTES + STAGING + VEC_BYTES + 256 + 1024;
  static constexpr int STAGES = (SMEM_BUDGET - FIXED) / B_STAGE > 6 ? 6 : (SMEM_BUDGET - FIXED) / B_STAGE;
  static constexpr int SMEM = FIXED + STAGES * B_STAGE;
  static_assert(STAGES >= 2 && SMEM <= SMEM_BUDGET, "shared memory budget");
  static_assert((B_STAGE / 2) % 1024 == 0, "half tiles must keep the 1024 B swizzle-atom alignment");
};

struct LnParams {
  const float* x;        // [M, 384] fp32 residual stream (read only)
  const float* gamma;    // [384]
  const float* beta;     // [384]
  const float* bias;     // [N]
  float eps;
  int M, N;
};

template <bool GELU, int BN>
__global__ void __launch_bounds__(LG_THREADS, 1)
gemm_ln_f16_wgmma_kernel(const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmC, int units,
                         LnParams p) {
  using Cfg = LnCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - raw);
  const uint32_t sA = base, sB = base + Cfg::A_BYTES, sOut = sB + STAGES * Cfg::B_STAGE;
  float* s_sum = reinterpret_cast<float*>(gbase + Cfg::A_BYTES + STAGES * Cfg::B_STAGE + Cfg::STAGING);
  float* s_rstd = s_sum + LG_BM;
  const RingBars<STAGES> bars{sOut + Cfg::STAGING + Cfg::VEC_BYTES};
  const uint32_t a_full = bars.base + 8u * (2 * STAGES), a_empty = a_full + 8u;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = (int)cluster_ctarank();
  const int cid = blockIdx.x >> 1, ncl = gridDim.x >> 1;
  const int tiles_n = p.N / BN;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmC);
    bars.init(4);   // the two MMA warp groups of both CTAs
    mbar_init(a_full, LG_LN_WARPS);
    mbar_init(a_empty, 2);
    mbar_fence_init();
  }
  __syncthreads();
  cluster_sync_all();

  if (warp < 4) {
    setmaxnreg_dec<56>();
    if (warp == 0) {
      const uint32_t ub = __shfl_sync(0xffffffffu, sB, 0);
      RingPos<STAGES> pos;
      for (int u = cid; u < units; u += ncl)
        for (int nt = 0; nt < tiles_n; ++nt)
          for (int kb = 0; kb < LG_SLABS; ++kb) {
            const int s = pos.slot;
            mbar_wait(bars.empty(s), pos.phase ^ 1u);
            if (elect_one()) {
              mbar_arrive_expect_tx(bars.full(s), Cfg::B_STAGE);
              tma_load_2d_mc(ub + s * Cfg::B_STAGE + rank * (Cfg::B_STAGE / 2), &tmB, bars.full(s), kb * BK,
                             nt * BN + rank * (BN / 2), (uint16_t)0x3);
            }
            __syncwarp();
            pos.advance();
          }
    } else {
      // ---- LayerNorm producers: warp w handles rows w-1, w+2, ... of the block
      const int lw = warp - 1;
      auto row_of = [&](int u) { return (2 * u + rank) * LG_BM; };
      auto stats = [&](int m0) {
        for (int r = lw; r < LG_BM; r += LG_LN_WARPS) {
          const int m = m0 + r;
          float S = 0.f, rstd = 0.f;
          if (m < p.M) {
            const float4* xr = reinterpret_cast<const float4*>(p.x + (long long)m * LG_K);
            float4 v[3];
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 3; ++i) {
              v[i] = xr[lane + 32 * i];
              s = __fadd_rn(s, ln_sum4(v[i]));
            }
            S = warp_sum(s);
            float q = 0.f;
#pragma unroll
            for (int i = 0; i < 3; ++i) q = __fadd_rn(q, ln_sq4(ln_center4(v[i], S, 1.0f / LG_K)));
            rstd = ln_rstd(warp_sum(q), 1.0f / LG_K, p.eps);
          }
          if (lane == 0) { s_sum[r] = S; s_rstd[r] = rstd; }
        }
        __syncwarp();
      };
      int lu = 0;
      if (cid < units) stats(row_of(cid));
      for (int u = cid; u < units; u += ncl, ++lu) {
        const int m0 = row_of(u);
        mbar_wait(a_empty, (lu & 1) ^ 1u);   // the MMA groups are done with the previous panel
        __syncwarp();
        for (int r = lw; r < LG_BM; r += LG_LN_WARPS) {
          const int m = m0 + r;
          const float S = s_sum[r], rstd = s_rstd[r];
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            const int c = 4 * (lane + 32 * i);   // first of this lane's 4 columns
            uint2 o = make_uint2(0u, 0u);        // rows past M: zeros (their outputs are clipped by the TMA store)
            if (m < p.M) {
              const float4 v = reinterpret_cast<const float4*>(p.x + (long long)m * LG_K)[lane + 32 * i];
              const float4 g = __ldg(reinterpret_cast<const float4*>(p.gamma) + lane + 32 * i);
              const float4 bt = __ldg(reinterpret_cast<const float4*>(p.beta) + lane + 32 * i);
              o = ln_out4(ln_center4(v, S, 1.0f / LG_K), rstd, g, bt);
            }
            const uint32_t addr = sw128_addr(sA + (c >> 6) * LG_SLAB_BYTES, r, (c & 63) >> 3) + (c & 7) * 2;
            asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(o.x), "r"(o.y) : "memory");
          }
        }
        fence_proxy_async_smem();   // generic-proxy panel writes -> visible to wgmma (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive(a_full);
        if (u + ncl < units) stats(row_of(u + ncl));   // overlaps this block's wgmmas
      }
    }
  } else {
    setmaxnreg_inc<224>();
    const int ct = threadIdx.x - 128;
    const int wg = ct >> 7, wi = (ct >> 5) & 3;
    const int fr = 64 * wg + 16 * wi + (lane >> 2), fc = 2 * (lane & 3);
    const bool issuer = ct == 0;
    const NamedBar<1, 256> epi_bar;
    RingPos<STAGES> pos;
    int cc = 0, lu = 0;
    float acc[BN / 2];
    auto mma = [&](int s, int kb) {
      mma_slab<BN>(acc, wgmma_desc_sw128(sA + kb * LG_SLAB_BYTES + wg * 64 * 128), wgmma_desc_sw128(sB + s * Cfg::B_STAGE),
                   kb == 0);
    };
    auto release = [&](int s) {
      mbar_arrive_cluster(bars.empty(s), 0);
      mbar_arrive_cluster(bars.empty(s), 1);
    };
    for (int u = cid; u < units; u += ncl, ++lu) {
      const int m0 = (2 * u + rank) * LG_BM;
      mbar_wait(a_full, lu & 1);
      for (int nt = 0; nt < tiles_n; ++nt) {
        const int last = consume_slabs(pos, bars, LG_SLABS, nullptr, mma, [&](int s) {
          if ((ct & 127) == 0) release(s);
        });
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
        if ((ct & 127) == 0) {
          release(last);
          if (nt == tiles_n - 1) mbar_arrive(a_empty);   // last reader of the panel: the next block may overwrite it
        }
        // ---- epilogue: 64-column boxes, fragments -> +bias (-> GELU) -> fp16 -> swizzled staging box -> TMA store
#pragma unroll
        for (int b = 0; b < BN / 64; ++b) {
          const int nc = nt * BN + b * 64;
          box_acquire(epi_bar, issuer);
          const uint32_t sbuf = sOut + (cc & 1) * LG_BOX_BYTES;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int ci = b * 8 + i;
            const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + nc + 8 * i + fc));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float x0 = acc[4 * ci + 2 * h] + bv.x, x1 = acc[4 * ci + 2 * h + 1] + bv.y;
              if constexpr (GELU) { x0 = gelu_erf(x0); x1 = gelu_erf(x1); }
              box_put_pair<true>(sbuf, fr + 8 * h, i, lane, x0, x1);
            }
          }
          box_issue(epi_bar, issuer, [&] { tma_store_2d(&tmC, sbuf, nc, m0); });
          ++cc;
        }
      }
    }
    if (issuer) tma_store_wait_all<0>();
  }
  cluster_pair_exit();
}

template <bool GELU, int BN>
static int launch_ln(const CUtensorMap& tmB, const CUtensorMap& tmC, const LnParams& p, cudaStream_t st, int kclass) {
  const int units = cdiv(cdiv(p.M, LG_BM), 2);   // pairs of row blocks
  return launch_cluster_pairs<gemm_ln_f16_wgmma_kernel<GELU, BN>, LnCfg<BN>::SMEM>(gemm_clusters(units), LG_THREADS, st,
                                                                                  kclass, tmB, tmC, units, p);
}

// tile width of the fused kernel for an N-column layer (0: not supported)
int gemm_ln_tile_n(int N) { return N % 192 == 0 ? 192 : (N % 128 == 0 ? 128 : 0); }

// tmB: weights [N, 384] f16 with box rows gemm_ln_tile_n(N) / 2; tmC: output [M, N] f16 (make_tmap_out)
int gemm_ln_f16_tc(const CUtensorMap& tmB, const CUtensorMap& tmC, const float* x, const float* gamma, const float* beta,
                   const float* bias, int M, int N, float eps, bool gelu, cudaStream_t st, int kclass) {
  DSS_REQUIRE(x && gamma && beta && bias, "gemm_ln: null pointer");
  DSS_REQUIRE(M > 0 && N > 0, "gemm_ln: empty problem");
  const int bn = gemm_ln_tile_n(N);
  DSS_REQUIRE(bn != 0, "gemm_ln: N = %d is not a multiple of 128", N);
  LnParams p{x, gamma, beta, bias, eps, M, N};
  if (bn == 192) return gelu ? launch_ln<true, 192>(tmB, tmC, p, st, kclass) : launch_ln<false, 192>(tmB, tmC, p, st, kclass);
  return gelu ? launch_ln<true, 128>(tmB, tmC, p, st, kclass) : launch_ln<false, 128>(tmB, tmC, p, st, kclass);
}

}  // namespace dss

using namespace dss;

extern "C" int dss_op_gemm_ln_f16(const float* x, const float* gamma, const float* beta, const void* Wt, const float* bias,
                                  void* out, int M, int N, int K, float eps, int gelu, dss_stream_t stream) {
  DSS_REQUIRE(K == LG_K, "gemm_ln: the fused LayerNorm GEMM is built for K = %d (ViT-S), got %d", LG_K, K);
  DSS_REQUIRE(Wt && out, "gemm_ln: null pointer");
  const int bn = gemm_ln_tile_n(N);
  DSS_REQUIRE(bn != 0, "gemm_ln: N = %d is not a multiple of 128", N);
  CUtensorMap tmB, tmC;
  int rc;
  if ((rc = make_tmap_f16(&tmB, Wt, N, K, bn / 2))) return rc;
  if ((rc = make_tmap_out(&tmC, out, M, N, 0))) return rc;
  return gemm_ln_f16_tc(tmB, tmC, x, gamma, beta, bias, M, N, eps, gelu != 0, static_cast<cudaStream_t>(stream), KC_GEMM_OTHER);
}
