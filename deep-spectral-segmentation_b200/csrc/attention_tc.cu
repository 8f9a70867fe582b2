// Multi-head attention (head dim 64) on the Hopper tensor cores: O = softmax(Q K^T / 8) V.
//
// One CTA per (128-query tile, head, image), two warp groups, each owning 64 query rows. Thread 0 drives the TMA: the
// Q tile and the K_j / V_j tiles come straight out of the packed qkv activations [B*T, 3d] (box 64 x 128, 128 B
// swizzle) through a 2-stage ring shared by both warp groups. Per key tile j, per warp group:
//   S = Q K^T    wgmma m64 x 128 x 16, x4, both operands K-major in shared memory        -> registers
//   online softmax in registers (row max / sum over the 4 lanes of a quad), P = 2^(s c - m c) packed to fp16 in the
//   register layout of the wgmma A operand: P never touches shared memory
//   O += P V     wgmma m64 x 64 x 16, x8, A = P from registers, B = V (MN-major: keys x head dims) -> registers
// Keys past T are masked to -inf; the output leaves through the (then free) Q tile with one 3-D TMA store (rows past T
// clipped per image).
#include <math.h>

#include "common.cuh"

namespace dss {

// one MUFU.EX2 (2 ulp), flushes denormal results to zero; exp2f would add range checks and fix-ups per element
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

constexpr int FA_BM = 128, FA_BN = 128, FA_D = 64, FA_THREADS = 256;
constexpr int FA_TILE = FA_BM * FA_D * 2;             // 16 KB: one [128 x 64] fp16 tile
constexpr int FA_KV_STAGES = 2;
// Q (reused as the output box) | K ring | V ring = 80 KB: two CTAs per SM
constexpr int FA_SMEM = FA_TILE * (1 + 2 * FA_KV_STAGES) + 1024;

__global__ void __launch_bounds__(FA_THREADS, 2)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmO, int T,
                       int heads) {
  extern __shared__ uint8_t fa_smem[];
  __shared__ __align__(8) uint64_t bars[1 + 2 * FA_KV_STAGES];
  const uint32_t raw = smem_u32(fa_smem);
  const uint32_t base = (raw + 1023u) & ~1023u;   // the 128 B swizzle pattern is a function of address bits [7,10)
  const uint32_t sQ = base, sK = base + FA_TILE, sV = sK + FA_KV_STAGES * FA_TILE;
  const uint32_t bar0 = smem_u32(bars);
  const uint32_t q_full = bar0;
  auto kv_full = [&](int s) { return bar0 + 8u * (1 + s); };
  auto kv_empty = [&](int s) { return bar0 + 8u * (1 + FA_KV_STAGES + s); };

  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = tid >> 7, wi = (tid >> 5) & 3;
  const int q0 = blockIdx.x * FA_BM, h = blockIdx.y, b = blockIdx.z;
  const int d = heads * FA_D;
  const int nt = (T + FA_BN - 1) / FA_BN;
  const int row0 = b * T;   // first row of this image in [B*T, 3d]

  auto load_kv = [&](int j) {
    const int s = j % FA_KV_STAGES;
    mbar_arrive_expect_tx(kv_full(s), 2 * FA_TILE);
    tma_load_2d(sK + s * FA_TILE, &tmQKV, kv_full(s), d + h * FA_D, row0 + j * FA_BN);
    tma_load_2d(sV + s * FA_TILE, &tmQKV, kv_full(s), 2 * d + h * FA_D, row0 + j * FA_BN);
  };
  if (tid == 0) {
    tma_prefetch_desc(&tmQKV);
    tma_prefetch_desc(&tmO);
    mbar_init(q_full, 1);
    for (int s = 0; s < FA_KV_STAGES; ++s) {
      mbar_init(kv_full(s), 1);
      mbar_init(kv_empty(s), 2);   // one arrival per warp group
    }
    mbar_fence_init();
    mbar_arrive_expect_tx(q_full, FA_TILE);
    tma_load_2d(sQ, &tmQKV, q_full, h * FA_D, row0 + q0);
    for (int j = 0; j < FA_KV_STAGES && j < nt; ++j) load_kv(j);
  }
  __syncthreads();

  // softmax in base 2: p = 2^(s c - m c), c = log2(e) / sqrt(64)
  const float sc = 1.4426950408889634f * 0.125f;
  const int fc = 2 * (lane & 3);                    // column of this thread inside an 8-column block
  float m_run[2] = {-INFINITY, -INFINITY};           // rows lane/4 and lane/4 + 8 of this warp's 16
  float l_run[2] = {0.f, 0.f};
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  const uint64_t qdesc = wgmma_desc_sw128(sQ + wg * 64 * 128);
  mbar_wait(q_full, 0);
  __syncwarp();

  for (int j = 0; j < nt; ++j) {
    const int s = j % FA_KV_STAGES;
    mbar_wait(kv_full(s), (j / FA_KV_STAGES) & 1);
    __syncwarp();   // wgmma is warp-aligned: reconverge after the per-thread barrier spin / thread 0's refill
    float sacc[64];
    const uint64_t kdesc = wgmma_desc_sw128(sK + s * FA_TILE);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < FA_D / 16; ++k) wgmma_m64n128_ss(sacc, qdesc + 2u * k, kdesc + 2u * k, k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(sacc);
    // mask keys beyond T (only the last tile can be partial)
    const int kbase = j * FA_BN;
    if (kbase + FA_BN > T) {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int key = kbase + 8 * i + fc;
        if (key >= T) sacc[4 * i] = sacc[4 * i + 2] = -INFINITY;
        if (key + 1 >= T) sacc[4 * i + 1] = sacc[4 * i + 3] = -INFINITY;
      }
    }
    float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
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
    // accumulator layout of two adjacent 8-key blocks == register A-operand layout of one 16-key step
    uint32_t pf[8][4];
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float p0 = ex2_approx(fmaf(sacc[4 * i], sc, -msc[0]));
      const float p1 = ex2_approx(fmaf(sacc[4 * i + 1], sc, -msc[0]));
      const float p2 = ex2_approx(fmaf(sacc[4 * i + 2], sc, -msc[1]));
      const float p3 = ex2_approx(fmaf(sacc[4 * i + 3], sc, -msc[1]));
      rs[0] += p0 + p1;
      rs[1] += p2 + p3;
      pf[i >> 1][(i & 1) * 2 + 0] = pack_half2(p0, p1);
      pf[i >> 1][(i & 1) * 2 + 1] = pack_half2(p2, p3);
    }
    l_run[0] += rs[0];
    l_run[1] += rs[1];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[4 * i] *= corr[0]; o[4 * i + 1] *= corr[0];
      o[4 * i + 2] *= corr[1]; o[4 * i + 3] *= corr[1];
    }
    const uint64_t vdesc = wgmma_desc_sw128(sV + s * FA_TILE);   // +16 key rows = +2048 B
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < FA_BN / 16; ++ks) wgmma_m64n64_rs_tb(o, pf[ks], vdesc + 128u * ks);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(o);
    // this warp group is done with K_j / V_j; thread 0 refills the slot once both groups are
    __syncwarp();
    if ((tid & 127) == 0) mbar_arrive(kv_empty(s));
    if (tid == 0 && j + FA_KV_STAGES < nt) {
      mbar_wait(kv_empty(s), (j / FA_KV_STAGES) & 1);
      load_kv(j + FA_KV_STAGES);
    }
  }

  // finalise: row sums across the 4 lanes of a quad, normalise, fp16 into this group's half of the Q tile (swizzled
  // as the output box), one TMA store of the 128 x 64 box
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const float inv0 = 1.0f / l_run[0], inv1 = 1.0f / l_run[1];
  const int r0 = 64 * wg + 16 * wi + (lane >> 2);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = r0 + 8 * hh;
      const float inv = hh ? inv1 : inv0;
      const uint32_t addr = sw128_addr(sQ, row, i) + (lane & 3) * 4;
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack_half2(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv))
                   : "memory");
    }
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (tid == 0) {
    tma_store_3d(&tmO, sQ, h * FA_D, q0, b);
    tma_store_commit();
    tma_store_wait_all<0>();
  }
}

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

}  // namespace dss

extern "C" int dss_op_attention_tc_f16(const void* qkv, void* out, int B, int T, int heads, dss_stream_t stream) {
  return dss::launch_attention_tc(qkv, out, B, T, heads, static_cast<cudaStream_t>(stream));
}
