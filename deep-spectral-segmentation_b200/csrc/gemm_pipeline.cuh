// The pipeline the persistent wgmma GEMM kernels of gemm.cu share (cooperative and ping-pong schedules): a ring of
// 64-deep K slabs filled by TMA and released by the MMA warp groups of both CTAs of a cluster pair, the wgmma k-steps
// of one slab, the 128 B-swizzled output staging box with its TMA store, and the cluster-pair launch. Each kernel keeps
// its own tile schedule, producer and epilogue arithmetic.
#pragma once
#include "common.cuh"

namespace dss {

constexpr int BK = 64, MMA_K = 16;     // K slab: one 128-byte swizzle atom of fp16 (one TMA box / 4 wgmma k-steps)
constexpr int SMEM_BUDGET = 232448;    // 227 KB of dynamic shared memory per block (sm_90)

#ifdef __CUDACC__

// Barrier block of a STAGES-slot ring at `base`: full[STAGES] | empty[STAGES]. A slot is full once the producer's
// expect_tx bytes have landed, and empty once `empty_count` consumer warp groups (counted over both CTAs of the pair)
// have released it.
template <int STAGES> struct RingBars {
  uint32_t base;
  __device__ __forceinline__ uint32_t full(int s) const { return base + 8u * s; }
  __device__ __forceinline__ uint32_t empty(int s) const { return base + 8u * (STAGES + s); }
  __device__ __forceinline__ void init(uint32_t empty_count) const {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), empty_count);
    }
  }
};

// Position in a STAGES-slot ring: the slot and the parity of the barrier phase it is in.
template <int STAGES> struct RingPos {
  int slot = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void advance() {
    if (++slot == STAGES) { slot = 0; phase ^= 1u; }
  }
  // n >= 0 slots at once
  __device__ __forceinline__ void skip(int n) {
    slot += n % STAGES;
    phase ^= (n / STAGES) & 1;
    if (slot >= STAGES) { slot -= STAGES; phase ^= 1u; }
  }
};

// The 4 wgmma k-steps of one K slab for H 64-row accumulators that share the B slab, interleaved per k-step. `first`:
// the tile's first slab, whose first k-step overwrites the accumulators.
template <int BN, int H>
__device__ __forceinline__ void mma_slab(float (&acc)[H][BN / 2], const uint64_t (&adesc)[H], uint64_t bdesc, bool first) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < BK / MMA_K; ++k)
#pragma unroll
    for (int h = 0; h < H; ++h) Wgmma<BN>::ss(acc[h], adesc[h] + 2u * k, bdesc + 2u * k, first && k == 0 ? 0u : 1u);
}
template <int BN>
__device__ __forceinline__ void mma_slab(float (&acc)[BN / 2], uint64_t adesc, uint64_t bdesc, bool first) {
  mma_slab<BN, 1>(*reinterpret_cast<float (*)[1][BN / 2]>(&acc), {adesc}, bdesc, first);
}

__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Consumer side of the ring for one tile of num_kb slabs. Per slab kb: wait until it has landed, issue its wgmmas
// (mma(slot, kb), which calls mma_slab) as one commit group, and once the previous group has retired (wgmma_wait<1>) hand that group's
// slot back (release(slot)). `stamp`, if not null, receives %globaltimer when the first slab has landed (phase trace).
// Returns the last slab's slot with its group still in flight: the caller retires it (wgmma_wait<0>) and releases it.
template <int STAGES, class Mma, class Release>
__device__ __forceinline__ int consume_slabs(RingPos<STAGES>& pos, const RingBars<STAGES>& bars, int num_kb,
                                             unsigned long long* stamp, Mma mma, Release release) {
  int prev = -1;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(bars.full(pos.slot), pos.phase);
    if (stamp != nullptr && kb == 0) *stamp = globaltimer();
    __syncwarp();   // wgmma is warp-aligned: reconverge after the per-thread barrier spin
    mma(pos.slot, kb);
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0) release(prev);
    prev = pos.slot;
    pos.advance();
  }
  return prev;
}

// Named barrier ID over THREADS threads. bar.sync is warp-aligned, so the warp reconverges first.
template <int ID, int THREADS> struct NamedBar {
  __device__ __forceinline__ void sync() const {
    __syncwarp();
    asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(THREADS) : "memory");
  }
};
// The same with the id chosen at run time: one barrier per warp group.
template <int THREADS> struct GroupBar {
  int id;
  __device__ __forceinline__ void sync() const {
    __syncwarp();
    asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(THREADS) : "memory");
  }
};

// ---- output staging box: 128 rows x 128 bytes (64 fp16 or 32 fp32 columns) in the 128 B-swizzled layout of the
// output tensor map, double buffered per group of epilogue threads, which share the named barrier `bar`.
// The box about to be written is free once the store issued from it two boxes ago has finished reading it.
template <class Bar>
__device__ __forceinline__ void box_acquire(const Bar& bar, bool issuer) {
  if (issuer) tma_store_wait_read<1>();
  bar.sync();
}
// One thread's accumulator pair: row `row`, columns 8 i + 2 (lane % 4) + {0, 1} of the box.
template <bool F16>
__device__ __forceinline__ void box_put_pair(uint32_t box, int row, int i, int lane, float x0, float x1) {
  if constexpr (F16) {
    const uint32_t addr = sw128_addr(box, row, i) + (lane & 3) * 4;
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack_half2(x0, x1)) : "memory");
  } else {
    const uint32_t addr = sw128_addr(box, row, 2 * i + ((lane & 3) >> 1)) + (lane & 1) * 8;
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(x0), "f"(x1) : "memory");
  }
}
// The written box goes to the TMA unit: the issuer's store() (TMA store or reduce-add of the box) in a bulk group.
template <class Bar, class Store>
__device__ __forceinline__ void box_issue(const Bar& bar, bool issuer, Store store) {
  fence_proxy_async_smem();   // generic-proxy smem writes -> visible to the TMA (async proxy)
  bar.sync();
  if (issuer) {
    store();
    tma_store_commit();
  }
}

// End of a cluster-pair kernel: the peer may still multicast / arrive into this CTA's shared memory until it is done too.
__device__ __forceinline__ void cluster_pair_exit() {
  __syncwarp();
  __syncthreads();
  cluster_sync_all();
}

#endif  // __CUDACC__

// ---- host side
// CTA pairs of a persistent launch over `items` work items: one CTA per SM
static inline int gemm_clusters(int items) {
  int sms = device_sm_count();
  if (sms <= 0) sms = 132;
  return items < sms / 2 ? items : sms / 2;
}

// Launches `kernel` on `clusters` clusters of two CTAs with SMEM bytes of dynamic shared memory (the attribute is set
// on the first launch of each kernel).
template <auto kernel, int SMEM, class... Args>
static int launch_cluster_pairs(int clusters, int threads, cudaStream_t st, int kclass, const Args&... args) {
  static bool attr_set = false;
  if (!attr_set) {
    DSS_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr_set = true;
  }
  LaunchScope scope(st, kclass);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(2 * clusters);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = SMEM;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  DSS_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, args...));
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}

}  // namespace dss
