// Segmentation evaluation counts (replace the pixel loops of the reference's semantic-segmentation/eval.py +
// eval_utils.get_iou and object-segmentation/main.py + metrics.compute_metrics).
//
// One device operation: a ragged batch of (prediction, target) uint8 label maps -> exact integer counts. Every output
// pixel (y, x) of image b reads the target at (top + y, left + x) and the prediction cell (rows[y], cols[x]) through
// host-built int32 gather tables. The tables express every nearest-neighbour resize and centre crop the reference
// applies, so the kernel does no floating-point index arithmetic. Pixels inside the top-left block (y < block_h,
// x < block_w) read the "inner" halves of the tables: the object app's downsample overwrites that block with a resize
// of the already-resized map, which no single separable table can express.
//
// Warps walk output rows (persistent grid, warp-granular stride). Semantic mode counts into a private shared-memory
// histogram per CTA with warp-aggregated increments (__match_any_sync: background dominates and would otherwise
// serialise the shared atomics), then adds its nonzero bins into the caller's int64 buffer with 64-bit integer atomics.
// Binary mode counts TP / FP / FN / TN per row with ballots. Integer arithmetic only: the counts do not depend on the
// batch or on scheduling.
#include <stdint.h>

#include <vector>

#include "common.cuh"

namespace dss {

constexpr int SE_THREADS = 256;
constexpr int SE_WARPS = SE_THREADS / 32;
constexpr int SE_MAX_BINS = 64;
constexpr int SE_MAX_WIDTH = 1 << 24;  // keeps one CTA round (SE_WARPS rows) far below 2^32 pixels

struct SegevalImage {
  long long pred_offset, target_offset, table_offset, row_start;
  int pred_w, target_w, top, left, h, w, block_h, block_w;
};

__device__ __forceinline__ int se_find_image(const SegevalImage* imgs, int B, long long row) {
  int lo = 0, hi = B - 1;  // last image whose row_start <= row
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (imgs[mid].row_start <= row) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Shared histogram [256][nbins] (uint32: the host sizes the grid so that no CTA sees 2^32 pixels).
template <bool BINARY>
__global__ void __launch_bounds__(SE_THREADS) segeval_kernel(const uint8_t* __restrict__ preds,
                                                             const uint8_t* __restrict__ targets,
                                                             const SegevalImage* __restrict__ imgs,
                                                             const int* __restrict__ tables, int B,
                                                             long long total_rows, int num_classes,
                                                             unsigned long long* __restrict__ counts) {
  extern __shared__ uint32_t hist[];
  const int nbins = num_classes + 1;
  const int lane = threadIdx.x & 31;
  if (!BINARY) {
    for (int i = threadIdx.x; i < 256 * nbins; i += SE_THREADS) hist[i] = 0;
    __syncthreads();
  }
  const long long warp0 = (long long)blockIdx.x * SE_WARPS + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * SE_WARPS;
  for (long long row = warp0; row < total_rows; row += nwarps) {
    const int b = se_find_image(imgs, B, row);
    const SegevalImage& im = imgs[b];  // a by-value copy spills 4 bytes in the semantic kernel
    const int y = (int)(row - im.row_start);
    const int* rt = tables + im.table_offset;  // rows_in[h], rows_out[h], cols_in[w], cols_out[w]
    const int* ct = rt + 2 * im.h;
    const bool row_in = y < im.block_h;
    const uint8_t* prow_in = preds + im.pred_offset + (long long)rt[y] * im.pred_w;
    const uint8_t* prow_out = preds + im.pred_offset + (long long)rt[im.h + y] * im.pred_w;
    const uint8_t* trow = targets + im.target_offset + (long long)(im.top + y) * im.target_w + im.left;
    uint32_t tp = 0, fp = 0, fn = 0, tn = 0;
    for (int x0 = 0; x0 < im.w; x0 += 32) {  // warp-uniform trip count: every lane reaches the match / ballot
      const int x = x0 + lane;
      const bool valid = x < im.w;
      int p = 0, t = 0;
      if (valid) {
        const bool in = row_in && x < im.block_w;
        p = in ? prow_in[ct[x]] : prow_out[ct[im.w + x]];
        t = trow[x];
      }
      if (BINARY) {
        const bool pp = p != 0, tt = t >= 128;
        tp += __popc(__ballot_sync(0xffffffffu, valid && pp && tt));
        fp += __popc(__ballot_sync(0xffffffffu, valid && pp && !tt));
        fn += __popc(__ballot_sync(0xffffffffu, valid && !pp && tt));
        tn += __popc(__ballot_sync(0xffffffffu, valid && !pp && !tt));
      } else {
        const bool use = valid && t != 255;
        const uint32_t key = use ? (uint32_t)(p * nbins + (t < num_classes ? t : num_classes)) : 0xffffffffu;
        const uint32_t peers = __match_any_sync(0xffffffffu, key);
        if (use && lane == __ffs(peers) - 1) atomicAdd(&hist[key], (uint32_t)__popc(peers));
      }
    }
    if (BINARY && lane == 0) {
      unsigned long long* o = counts + 4 * (long long)b;
      if (tp) atomicAdd(o + 0, (unsigned long long)tp);
      if (fp) atomicAdd(o + 1, (unsigned long long)fp);
      if (fn) atomicAdd(o + 2, (unsigned long long)fn);
      if (tn) atomicAdd(o + 3, (unsigned long long)tn);
    }
  }
  if (!BINARY) {
    __syncthreads();
    for (int i = threadIdx.x; i < 256 * nbins; i += SE_THREADS)
      if (hist[i]) atomicAdd(counts + i, (unsigned long long)hist[i]);
  }
}

}  // namespace dss

using namespace dss;

extern "C" size_t dss_segeval_workspace_bytes(int B, long long table_entries) {
  if (B <= 0 || table_entries < 0) return 0;
  return align_up((size_t)B * sizeof(SegevalImage), 256) + align_up((size_t)table_entries * sizeof(int), 256);
}

extern "C" int dss_segeval_counts(const uint8_t* preds, long long preds_bytes, const uint8_t* targets,
                                  long long targets_bytes, const long long* images_host, int B, const int* tables_host,
                                  long long table_entries, int mode, int num_classes, long long* counts, void* ws,
                                  size_t ws_bytes, dss_stream_t stream) {
  DSS_REQUIRE(preds && targets && images_host && tables_host && counts && ws, "segeval_counts: null pointer");
  DSS_REQUIRE(B > 0 && table_entries >= 0 && preds_bytes >= 0 && targets_bytes >= 0,
              "segeval_counts: bad batch (B=%d, %lld table entries)", B, table_entries);
  DSS_REQUIRE(mode == DSS_SEGEVAL_SEMANTIC || mode == DSS_SEGEVAL_BINARY, "segeval_counts: unknown mode %d", mode);
  if (mode == DSS_SEGEVAL_SEMANTIC && (num_classes < 1 || num_classes + 1 > SE_MAX_BINS)) {
    set_error("segeval_counts: num_classes + 1 = %d target bins (1 < bins <= %d: one CTA holds 256 x bins counts in "
              "shared memory)", num_classes + 1, SE_MAX_BINS);
    return DSS_ERR_UNSUPPORTED;
  }
  if (ws_bytes < dss_segeval_workspace_bytes(B, table_entries)) {
    set_error("segeval_counts: workspace too small (%zu < %zu)", ws_bytes,
              dss_segeval_workspace_bytes(B, table_entries));
    return DSS_ERR_WORKSPACE;
  }
  std::vector<SegevalImage> imgs(B);
  long long rows = 0, max_w = 0;
  for (int b = 0; b < B; ++b) {
    const long long* d = images_host + DSS_SEGEVAL_FIELDS * b;
    const long long po = d[0], ph = d[1], pw = d[2], to = d[3], th = d[4], tw = d[5], top = d[6], left = d[7];
    const long long h = d[8], w = d[9], bh = d[10], bw = d[11], tab = d[12];
    DSS_REQUIRE(ph > 0 && pw > 0 && th > 0 && tw > 0 && h > 0 && w > 0, "segeval_counts: image %d has an empty map",
                b);
    if (ph * pw >= (1ll << 31) || th * tw >= (1ll << 31) || w > SE_MAX_WIDTH) {
      set_error("segeval_counts: image %d: maps of 2^31 cells or rows wider than %d are not supported", b,
                SE_MAX_WIDTH);
      return DSS_ERR_UNSUPPORTED;
    }
    if (po < 0 || po + ph * pw > preds_bytes || to < 0 || to + th * tw > targets_bytes) {
      set_error("segeval_counts: image %d reads outside the prediction / target buffers", b);
      return DSS_ERR_UNSUPPORTED;
    }
    if (top < 0 || left < 0 || top + h > th || left + w > tw || bh < 0 || bw < 0) {
      set_error("segeval_counts: image %d: crop (%lld, %lld, %lld x %lld) outside its %lld x %lld target", b, top,
                left, h, w, th, tw);
      return DSS_ERR_UNSUPPORTED;
    }
    if (tab < 0 || tab + 2 * (h + w) > table_entries) {
      set_error("segeval_counts: image %d: gather tables outside the %lld table entries", b, table_entries);
      return DSS_ERR_UNSUPPORTED;
    }
    const int* t = tables_host + tab;
    for (long long i = 0; i < 2 * (h + w); ++i) {
      const long long lim = i < 2 * h ? ph : pw;
      if (t[i] < 0 || t[i] >= lim) {
        set_error("segeval_counts: image %d: gather table entry %lld = %d outside the %lld x %lld prediction", b, i,
                  t[i], ph, pw);
        return DSS_ERR_UNSUPPORTED;
      }
    }
    imgs[b] = SegevalImage{po, to, tab, rows, (int)pw, (int)tw, (int)top, (int)left, (int)h, (int)w,
                           (int)(bh < h ? bh : h), (int)(bw < w ? bw : w)};
    rows += h;
    if (w > max_w) max_w = w;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t img_bytes = align_up((size_t)B * sizeof(SegevalImage), 256);
  int* d_tables = reinterpret_cast<int*>(static_cast<char*>(ws) + img_bytes);
  // pageable sources: the copies are staged before cudaMemcpyAsync returns, so `imgs` may go out of scope
  DSS_CHECK_CUDA(cudaMemcpyAsync(ws, imgs.data(), (size_t)B * sizeof(SegevalImage), cudaMemcpyHostToDevice, st));
  if (table_entries > 0)
    DSS_CHECK_CUDA(cudaMemcpyAsync(d_tables, tables_host, (size_t)table_entries * sizeof(int), cudaMemcpyHostToDevice,
                                   st));
  unsigned long long* out = reinterpret_cast<unsigned long long*>(counts);
  if (mode == DSS_SEGEVAL_BINARY) DSS_CHECK_CUDA(cudaMemsetAsync(out, 0, (size_t)B * 4 * sizeof(long long), st));

  // Two CTAs per SM, more if one CTA would otherwise walk 2^32 pixels (its uint32 histogram would wrap): a warp takes
  // at most ceil(rows / warps) rows of at most max_w pixels.
  long long grid = 2ll * device_sm_count();
  while (grid < rows &&
         (long long)SE_WARPS * ((rows + grid * SE_WARPS - 1) / (grid * SE_WARPS)) * max_w >= (1ll << 32))
    grid *= 2;
  if (grid > rows) grid = rows;
  const SegevalImage* d_imgs = reinterpret_cast<const SegevalImage*>(ws);
  LaunchScope scope(st, KC_MISC);
  if (mode == DSS_SEGEVAL_BINARY) {
    segeval_kernel<true><<<(unsigned)grid, SE_THREADS, 0, st>>>(preds, targets, d_imgs, d_tables, B, rows, 0, out);
  } else {
    const size_t smem = (size_t)256 * (num_classes + 1) * sizeof(uint32_t);
    DSS_CHECK_CUDA(cudaFuncSetAttribute(segeval_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)smem));
    segeval_kernel<false><<<(unsigned)grid, SE_THREADS, smem, st>>>(preds, targets, d_imgs, d_tables, B, rows,
                                                                      num_classes, out);
  }
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}
