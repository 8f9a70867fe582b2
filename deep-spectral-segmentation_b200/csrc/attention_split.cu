// Multi-head attention (head dim 64) at fp32-equivalent accuracy on the fp16 tensor cores: the attention of
// DSS_VIT_PRECISION_FP32. Operands come from qkv_split_kernel (vit_split.cu), per head 192 columns of [B*T, 9d]:
//   Q' = [qhi | qhi/64 | 64 qlo]   K' = [khi | 64 klo | khi/64]   V' = [vhi | 64 vlo | vhi/64]
// so that S = Q' K'^T over K = 192 is qhi khi + qhi klo + qlo khi (12 k-steps), and with P = Phi + Plo split in registers
//   O += Phi Vhi + (Phi/64)(64 Vlo) + (64 Plo)(Vhi/64)          (three m64n64k16 passes of 4 k-steps per key tile)
// Softmax and the running row max / sum are fp32 (the row sum adds the unsplit fp32 p).
//
// One CTA per (128-query tile, head, image), two warp groups of 64 query rows, thread 0 drives the TMA, as
// attention_wgmma_kernel. Tiling: Q' is 128 x 192 fp16 = 48 KB; a 128-key K'/V' stage would be 96 KB, so two stages
// would not fit beside Q' (240 KB > 227 KB). 64-key stages (K' and V' 24 KB each) give a two-stage ring in 144 KB: one
// CTA per SM, the next tile's load under the current tile's MMAs. The output (normalised O, split in A order
// [hi | hi/64 | 64 lo], each group d wide, head h at columns h*64 of each group) is the proj GEMM's A operand and is
// stored straight from registers (rows past T skipped).
#include <math.h>

#include "common.cuh"

namespace dss {

constexpr int AS_BM = 128, AS_BN = 64, AS_THREADS = 256, AS_STAGES = 2;
constexpr int AS_BOX = 64 * 64 * 2;                    // 8 KB: one 64-row x 64-column fp16 TMA box
constexpr int AS_Q = 3 * 2 * AS_BOX;                   // Q': 3 groups x 128 rows
constexpr int AS_KV = 3 * AS_BOX;                      // one K' or V' stage: 3 groups x 64 keys
constexpr int AS_SMEM = AS_Q + 2 * AS_STAGES * AS_KV + 1024;

__device__ __forceinline__ float as_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

#define AS_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                   "+f"(d[i + 6]), "+f"(d[i + 7])
// D[64 x 64] (+)= A(smem) * B(smem), both K-major
__device__ __forceinline__ void wgmma_m64n64_ss(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : AS_ACC8(0), AS_ACC8(8), AS_ACC8(16), AS_ACC8(24)
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
#undef AS_ACC8

__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
  __half2 h = __halves2half2(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __launch_bounds__(AS_THREADS, 1)
attention_split_kernel(const __grid_constant__ CUtensorMap tmQKV, __half* __restrict__ out, int T, int heads) {
  extern __shared__ uint8_t as_smem[];
  __shared__ __align__(8) uint64_t bars[1 + 2 * AS_STAGES];
  const uint32_t base = (smem_u32(as_smem) + 1023u) & ~1023u;
  const uint32_t sQ = base, sK = base + AS_Q, sV = sK + AS_STAGES * AS_KV;
  const uint32_t bar0 = smem_u32(bars);
  const uint32_t q_full = bar0;
  auto kv_full = [&](int s) { return bar0 + 8u * (1 + s); };
  auto kv_empty = [&](int s) { return bar0 + 8u * (1 + AS_STAGES + s); };

  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = tid >> 7, wi = (tid >> 5) & 3;
  const int q0 = blockIdx.x * AS_BM, h = blockIdx.y, b = blockIdx.z;
  const int d = heads * 64;
  const int nt = (T + AS_BN - 1) / AS_BN;
  const int row0 = b * T;

  auto load_kv = [&](int j) {
    const int s = j % AS_STAGES;
    mbar_arrive_expect_tx(kv_full(s), 2 * AS_KV);
    for (int g = 0; g < 3; ++g) {
      tma_load_2d(sK + s * AS_KV + g * AS_BOX, &tmQKV, kv_full(s), 3 * d + h * 192 + g * 64, row0 + j * AS_BN);
      tma_load_2d(sV + s * AS_KV + g * AS_BOX, &tmQKV, kv_full(s), 6 * d + h * 192 + g * 64, row0 + j * AS_BN);
    }
  };
  if (tid == 0) {
    tma_prefetch_desc(&tmQKV);
    mbar_init(q_full, 1);
    for (int s = 0; s < AS_STAGES; ++s) {
      mbar_init(kv_full(s), 1);
      mbar_init(kv_empty(s), 2);   // one arrival per warp group
    }
    mbar_fence_init();
    mbar_arrive_expect_tx(q_full, AS_Q);
    // Q' group g: rows 0-63 at +0, rows 64-127 at +8 KB, so each group is one 128-row swizzled tile
    for (int g = 0; g < 3; ++g)
      for (int half = 0; half < 2; ++half)
        tma_load_2d(sQ + (2 * g + half) * AS_BOX, &tmQKV, q_full, h * 192 + g * 64, row0 + q0 + 64 * half);
    for (int j = 0; j < AS_STAGES && j < nt; ++j) load_kv(j);
  }
  __syncthreads();

  const float sc = 1.4426950408889634f * 0.125f;   // softmax in base 2: p = 2^(s c - m c)
  const int fc = 2 * (lane & 3);
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  mbar_wait(q_full, 0);
  __syncwarp();

  for (int j = 0; j < nt; ++j) {
    const int s = j % AS_STAGES;
    mbar_wait(kv_full(s), (j / AS_STAGES) & 1);
    __syncwarp();
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
    const int kbase = j * AS_BN;
    if (kbase + AS_BN > T) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int key = kbase + 8 * i + fc;
        if (key >= T) sacc[4 * i] = sacc[4 * i + 2] = -INFINITY;
        if (key + 1 >= T) sacc[4 * i + 1] = sacc[4 * i + 3] = -INFINITY;
      }
    }
    float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      mx[0] = fmaxf(mx[0], fmaxf(sacc[4 * i], sacc[4 * i + 1]));
      mx[1] = fmaxf(mx[1], fmaxf(sacc[4 * i + 2], sacc[4 * i + 3]));
    }
    float corr[2], msc[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      corr[r] = as_ex2((m_run[r] - mx[r]) * sc);
      m_run[r] = mx[r];
      msc[r] = mx[r] * sc;
      l_run[r] *= corr[r];
    }
    // P in the register A-operand layout (two adjacent 8-key blocks = one 16-key step), split into its three groups
    uint32_t p_hi[4][4], p_his[4][4], p_los[4][4];
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float p[4];
      p[0] = as_ex2(fmaf(sacc[4 * i], sc, -msc[0]));
      p[1] = as_ex2(fmaf(sacc[4 * i + 1], sc, -msc[0]));
      p[2] = as_ex2(fmaf(sacc[4 * i + 2], sc, -msc[1]));
      p[3] = as_ex2(fmaf(sacc[4 * i + 3], sc, -msc[1]));
      rs[0] += p[0] + p[1];
      rs[1] += p[2] + p[3];
      SplitF16 sp[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) sp[t] = split_f16(p[t]);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        p_hi[i >> 1][(i & 1) * 2 + r] = pack_h2(sp[2 * r].hi, sp[2 * r + 1].hi);
        p_his[i >> 1][(i & 1) * 2 + r] = pack_h2(sp[2 * r].hi_s, sp[2 * r + 1].hi_s);
        p_los[i >> 1][(i & 1) * 2 + r] = pack_h2(sp[2 * r].lo_s, sp[2 * r + 1].lo_s);
      }
    }
    l_run[0] += rs[0];
    l_run[1] += rs[1];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[4 * i] *= corr[0]; o[4 * i + 1] *= corr[0];
      o[4 * i + 2] *= corr[1]; o[4 * i + 3] *= corr[1];
    }
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
    __syncwarp();
    if ((tid & 127) == 0) mbar_arrive(kv_empty(s));
    if (tid == 0 && j + AS_STAGES < nt) {
      mbar_wait(kv_empty(s), (j / AS_STAGES) & 1);
      load_kv(j + AS_STAGES);
    }
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
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
      *reinterpret_cast<uint32_t*>(orow + 8 * i) = pack_h2(a.hi, c.hi);
      *reinterpret_cast<uint32_t*>(orow + d + 8 * i) = pack_h2(a.hi_s, c.hi_s);
      *reinterpret_cast<uint32_t*>(orow + 2 * d + 8 * i) = pack_h2(a.lo_s, c.lo_s);
    }
  }
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

}  // namespace dss

extern "C" int dss_op_attention_split_f16(const float* qkv, void* qkv_split, void* out, int B, int T, int heads,
                                          dss_stream_t stream) {
  DSS_REQUIRE(qkv, "attention_split: null pointer");
  DSS_REQUIRE(B > 0 && T > 0 && heads > 0, "attention_split: empty problem");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = dss::launch_qkv_split(qkv, qkv_split, (long long)B * T, heads * 64, st);
  if (rc) return rc;
  return dss::launch_attention_split(qkv_split, out, B, T, heads, st);
}
