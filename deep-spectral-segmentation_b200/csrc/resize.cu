// Pillow's Image.resize((W_out, H_out), Image.BILINEAR) of a batch of uint8 RGB images of one size, bit for bit
// (the low-resolution colour image of the reference's extract/extract.py:199-204).
//
// Pillow resizes in two integer passes: horizontal, then vertical over the horizontal pass's uint8 result. Each output
// index o of an axis reads the window [first_o, first_o + count_o) of its input with fixed-point weights (22 fractional
// bits) that the host builds per (input size, output size) pair (resize.py restates Pillow's double-precision window
// and weight arithmetic). Every sum starts at 2^21 (round half up) and is clipped to [0, 255] after the shift.
//
// One thread per output pixel, three channels each: for every row of its vertical window it recomputes the horizontal
// pass of that row at its own column, clips it to uint8 and accumulates it with the row's vertical weight. Bilinear
// windows overlap about twice, so each intermediate value is computed about twice, and no intermediate image or
// per-call scratch beyond the tables is needed. The arithmetic is Pillow's int32 arithmetic, in Pillow's order.
#include <stdint.h>

#include <vector>

#include "common.cuh"

namespace dss {

constexpr int RS_THREADS = 128;
constexpr int RS_BITS = 22;

__device__ __forceinline__ int rs_clip8(int acc) {
  if (acc >= (1 << RS_BITS << 8)) return 255;
  if (acc <= 0) return 0;
  return acc >> RS_BITS;
}

// bounds_*: {first, count} per output index; weights_*: taps per output index (zero past count).
// unit (UNIT_F32): the 256 values float(v / 255.0), built on the host in double.
template <bool UNIT_F32>
__global__ void __launch_bounds__(RS_THREADS) resize_bilinear_kernel(const uint8_t* __restrict__ in, int H, int W,
                                                                     int H_out, int W_out,
                                                                     const int* __restrict__ bounds_y,
                                                                     const int* __restrict__ weights_y, int taps_y,
                                                                     const int* __restrict__ bounds_x,
                                                                     const int* __restrict__ weights_x, int taps_x,
                                                                     const float* __restrict__ unit,
                                                                     void* __restrict__ out) {
  __shared__ float s_unit[UNIT_F32 ? 256 : 1];
  if (UNIT_F32) {
    for (int i = threadIdx.x; i < 256; i += RS_THREADS) s_unit[i] = unit[i];
    __syncthreads();
  }
  const int xo = blockIdx.x * RS_THREADS + threadIdx.x;
  if (xo >= W_out) return;
  const int yo = blockIdx.y, b = blockIdx.z;
  const int y0 = bounds_y[2 * yo], ny = bounds_y[2 * yo + 1];
  const int x0 = bounds_x[2 * xo], nx = bounds_x[2 * xo + 1];
  const int* ky = weights_y + (size_t)yo * taps_y;
  const int* kx = weights_x + (size_t)xo * taps_x;
  const uint8_t* src = in + ((size_t)b * H + y0) * W * 3 + (size_t)x0 * 3;
  int a0 = 1 << (RS_BITS - 1), a1 = a0, a2 = a0;
  for (int y = 0; y < ny; ++y, src += (size_t)W * 3) {
    int h0 = 1 << (RS_BITS - 1), h1 = h0, h2 = h0;
    for (int x = 0; x < nx; ++x) {
      const int k = __ldg(kx + x);
      h0 += (int)__ldg(src + 3 * x) * k;
      h1 += (int)__ldg(src + 3 * x + 1) * k;
      h2 += (int)__ldg(src + 3 * x + 2) * k;
    }
    const int k = __ldg(ky + y);
    a0 += rs_clip8(h0) * k;
    a1 += rs_clip8(h1) * k;
    a2 += rs_clip8(h2) * k;
  }
  const size_t o = (((size_t)b * H_out + yo) * W_out + xo) * 3;
  if (UNIT_F32) {
    float* dst = static_cast<float*>(out) + o;
    dst[0] = s_unit[rs_clip8(a0)];
    dst[1] = s_unit[rs_clip8(a1)];
    dst[2] = s_unit[rs_clip8(a2)];
  } else {
    uint8_t* dst = static_cast<uint8_t*>(out) + o;
    dst[0] = (uint8_t)rs_clip8(a0);
    dst[1] = (uint8_t)rs_clip8(a1);
    dst[2] = (uint8_t)rs_clip8(a2);
  }
}

// Workspace layout: bounds_y [2 H_out], bounds_x [2 W_out], weights_y [H_out taps_y], weights_x [W_out taps_x] int32,
// unit [256] fp32, each 256-byte aligned.
static size_t rs_part(size_t n) { return align_up(n * 4, 256); }

static bool rs_check_axis(const int* bounds, const int* weights, int out, int taps, int in, const char* axis) {
  for (int o = 0; o < out; ++o) {
    const int first = bounds[2 * o], count = bounds[2 * o + 1];
    if (first < 0 || count < 1 || count > taps || first + count > in) {
      set_error("resize_bilinear: %s window %d = {%d, %d} outside the %d input pixels or its %d taps", axis, o, first,
                count, in, taps);
      return false;
    }
    for (int t = 0; t < taps; ++t) {
      if (weights[(size_t)o * taps + t] < 0 || weights[(size_t)o * taps + t] > (1 << RS_BITS)) {
        set_error("resize_bilinear: %s weight [%d, %d] = %d outside [0, 2^22]", axis, o, t,
                  weights[(size_t)o * taps + t]);
        return false;
      }
    }
  }
  return true;
}

}  // namespace dss

using namespace dss;

extern "C" size_t dss_resize_workspace_bytes(int H_out, int W_out, int taps_y, int taps_x) {
  if (H_out <= 0 || W_out <= 0 || taps_y <= 0 || taps_x <= 0) return 0;
  return rs_part(2 * (size_t)H_out) + rs_part(2 * (size_t)W_out) + rs_part((size_t)H_out * taps_y) +
         rs_part((size_t)W_out * taps_x) + rs_part(256);
}

extern "C" int dss_resize_bilinear(const uint8_t* images, int B, int H, int W, int H_out, int W_out,
                                   const int* bounds_y_host, const int* weights_y_host, int taps_y,
                                   const int* bounds_x_host, const int* weights_x_host, int taps_x, int kind, void* out,
                                   void* ws, size_t ws_bytes, dss_stream_t stream) {
  DSS_REQUIRE(images && bounds_y_host && weights_y_host && bounds_x_host && weights_x_host && out && ws,
              "resize_bilinear: null pointer");
  DSS_REQUIRE(B > 0 && H > 0 && W > 0 && H_out > 0 && W_out > 0 && taps_y > 0 && taps_x > 0,
              "resize_bilinear: empty problem (B=%d, %d x %d -> %d x %d, taps %d / %d)", B, H, W, H_out, W_out, taps_y,
              taps_x);
  DSS_REQUIRE(H_out <= H && W_out <= W, "resize_bilinear: output %d x %d larger than the input %d x %d (downscaling only)",
              H_out, W_out, H, W);
  DSS_REQUIRE(kind == DSS_RESIZE_U8 || kind == DSS_RESIZE_UNIT_F32, "resize_bilinear: unknown output kind %d", kind);
  if (B > 65535 || H_out > 65535) {
    set_error("resize_bilinear: B = %d or H_out = %d past the grid limit 65535", B, H_out);
    return DSS_ERR_UNSUPPORTED;
  }
  if (ws_bytes < dss_resize_workspace_bytes(H_out, W_out, taps_y, taps_x)) {
    set_error("resize_bilinear: workspace too small (%zu < %zu)", ws_bytes,
              dss_resize_workspace_bytes(H_out, W_out, taps_y, taps_x));
    return DSS_ERR_WORKSPACE;
  }
  if (!rs_check_axis(bounds_y_host, weights_y_host, H_out, taps_y, H, "vertical") ||
      !rs_check_axis(bounds_x_host, weights_x_host, W_out, taps_x, W, "horizontal"))
    return DSS_ERR_BAD_ARG;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  char* p = static_cast<char*>(ws);
  int* by = reinterpret_cast<int*>(p);
  int* bx = reinterpret_cast<int*>(p += rs_part(2 * (size_t)H_out));
  int* wy = reinterpret_cast<int*>(p += rs_part(2 * (size_t)W_out));
  int* wx = reinterpret_cast<int*>(p += rs_part((size_t)H_out * taps_y));
  float* unit = reinterpret_cast<float*>(p += rs_part((size_t)W_out * taps_x));
  // pageable sources: the copies are staged before cudaMemcpyAsync returns
  DSS_CHECK_CUDA(cudaMemcpyAsync(by, bounds_y_host, 2 * (size_t)H_out * 4, cudaMemcpyHostToDevice, st));
  DSS_CHECK_CUDA(cudaMemcpyAsync(bx, bounds_x_host, 2 * (size_t)W_out * 4, cudaMemcpyHostToDevice, st));
  DSS_CHECK_CUDA(cudaMemcpyAsync(wy, weights_y_host, (size_t)H_out * taps_y * 4, cudaMemcpyHostToDevice, st));
  DSS_CHECK_CUDA(cudaMemcpyAsync(wx, weights_x_host, (size_t)W_out * taps_x * 4, cudaMemcpyHostToDevice, st));
  const dim3 grid(cdiv(W_out, RS_THREADS), H_out, B);
  LaunchScope scope(st, KC_MISC);
  if (kind == DSS_RESIZE_UNIT_F32) {
    // numpy's (v / 255.0).astype(np.float32): a double division, then one rounding to float
    std::vector<float> table(256);
    for (int v = 0; v < 256; ++v) table[v] = (float)((double)v / 255.0);
    DSS_CHECK_CUDA(cudaMemcpyAsync(unit, table.data(), 256 * sizeof(float), cudaMemcpyHostToDevice, st));
    resize_bilinear_kernel<true><<<grid, RS_THREADS, 0, st>>>(images, H, W, H_out, W_out, by, wy, taps_y, bx, wx,
                                                                taps_x, unit, out);
  } else {
    resize_bilinear_kernel<false><<<grid, RS_THREADS, 0, st>>>(images, H, W, H_out, W_out, by, wy, taps_y, bx, wx,
                                                                 taps_x, unit, out);
  }
  DSS_CHECK_CUDA(cudaGetLastError());
  return DSS_OK;
}
