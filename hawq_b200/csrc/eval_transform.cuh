// The reference's evaluation transform on the device (quant_train.py:427-438, tvm_benchmark/test_resnet_accuracy_imagenet.py:82-90):
// Resize(S) -> CenterCrop(Ch, Cw) -> ToTensor -> Normalize -> QuantAct input branch, from a ragged batch of uint8 HWC RGB images of
// any size to the int8 NHWC network input [B, Ch, Cw, 3], in one launch.
//
// The resize is PIL's bilinear ImagingResample for 8-bit images (torchvision.transforms.Resize on PIL images), restated exactly:
// per output sample a window of source samples and fixed-point coefficients (PRECISION_BITS 22) computed from double-precision
// weights, the horizontal pass first, each pass rounded back to uint8.  Every double operation is one IEEE operation (__d*_rn: nvcc
// would otherwise contract a * b + c into an FMA) and every (int) truncates, as in the C source.  Only the crop is computed: the
// resized image is never materialised.
//
// One CTA per (32 crop columns, 16 crop rows, image).  Everything per image (resized size, crop offsets, windows, coefficients)
// is derived here from the image's hawq_image_desc, so the grid depends only on B, Ch and Cw and one captured graph serves any
// image sizes.  The CTA streams the source rows its output rows need through shared memory, ET_CHUNK at a time: the horizontal
// pass (only the tile's columns) rounds them to uint8 in shared memory, the vertical pass accumulates them in int32 registers.
// Shared memory is fixed: with S >= ET_MIN_RESIZE and sides <= ET_MAX_SIDE a pass downsizes by at most 64, so a window has at
// most ET_MAX_TAPS = 129 taps.
#pragma once
#include "common.cuh"
#include "elementwise.cuh"

namespace hawq {

constexpr int ET_TW = 32, ET_TR = 16, ET_CHUNK = 16;          // crop columns and rows per CTA, source rows per streamed chunk
constexpr int ET_ELEMS = ET_TW * 3;                           // (column, channel) pairs of one tile row
constexpr int ET_THREADS = 2 * ET_ELEMS;                      // two threads per pair, each owning half of the tile's rows
constexpr int ET_ROWS_PER_THREAD = ET_TR / 2;
constexpr int ET_MAX_SIDE = 16384, ET_MIN_RESIZE = 256, ET_MAX_TAPS = 129;
constexpr int ET_PRECISION_BITS = 22;

// One pass from `in` to `out` samples (PIL precompute_coeffs, bilinear: support 1.0 * filterscale).
struct EtPass {
  double scale, support, ss;
  int in;
};

__device__ __forceinline__ EtPass et_pass(int in, int out) {
  EtPass p;
  p.scale = __ddiv_rn((double)in, (double)out);
  p.support = fmax(p.scale, 1.0);                             // filterscale; support = 1.0 * filterscale
  p.ss = __ddiv_rn(1.0, p.support);
  p.in = in;
  return p;
}

__device__ __forceinline__ double et_tri(const EtPass& p, int x, double center) {
  double t = fabs(__dmul_rn(__dadd_rn(__dsub_rn((double)x, center), 0.5), p.ss));
  return t < 1.0 ? __dsub_rn(1.0, t) : 0.0;
}

// Window of output sample xx: writes its coefficients to k[0, n) and returns (xmin, n).
__device__ __forceinline__ int2 et_window(const EtPass& p, int xx, int* k) {
  const double center = __dmul_rn(__dadd_rn((double)xx, 0.5), p.scale);
  const int xmin = max((int)__dadd_rn(__dsub_rn(center, p.support), 0.5), 0);
  const int n = min(min((int)__dadd_rn(__dadd_rn(center, p.support), 0.5), p.in) - xmin, ET_MAX_TAPS);
  double ww = 0.0;
  for (int i = 0; i < n; ++i) ww = __dadd_rn(ww, et_tri(p, i + xmin, center));
  for (int i = 0; i < n; ++i) {
    double w = et_tri(p, i + xmin, center);
    if (ww != 0.0) w = __ddiv_rn(w, ww);
    const double s = __dmul_rn(w, (double)(1 << ET_PRECISION_BITS));
    k[i] = w < 0.0 ? (int)__dadd_rn(-0.5, s) : (int)__dadd_rn(0.5, s);
  }
  return make_int2(xmin, n);
}

__device__ __forceinline__ int et_clip8(int v) { return min(max(v >> ET_PRECISION_BITS, 0), 255); }

__global__ void __launch_bounds__(ET_THREADS) resize_crop_quantize_u8_kernel(
    const uint8_t* __restrict__ pixels, long long pixel_bytes, const hawq_image_desc* __restrict__ table, int S, int Ch, int Cw,
    float m0, float m1, float m2, float s0, float s1, float s2, float inv_scale, int lo, int hi, int8_t* __restrict__ out) {
  __shared__ int8_t lut[3 * 256];
  __shared__ int kh[ET_TW][ET_MAX_TAPS];
  __shared__ int kv[ET_TR][ET_MAX_TAPS];
  __shared__ int2 win_h[ET_TW], win_v[ET_TR];
  __shared__ uint8_t rows[ET_CHUNK][ET_ELEMS];

  const int tid = threadIdx.x, b = blockIdx.z;
  const int ox0 = blockIdx.x * ET_TW, oy0 = blockIdx.y * ET_TR;
  const int tw = min(ET_TW, Cw - ox0), tr = min(ET_TR, Ch - oy0);
  build_input_lut(lut, m0, m1, m2, s0, s1, s2, inv_scale, lo, hi);

  // an absent slot (h == 0), or an entry that does not describe an image inside the arena, yields the zero pixel's value
  const hawq_image_desc d = table[b];
  const bool present = d.h >= 1 && d.w >= 1 && d.h <= ET_MAX_SIDE && d.w <= ET_MAX_SIDE && d.offset >= 0 &&
                       d.offset <= pixel_bytes - 3LL * d.h * d.w;
  if (present) {
    // torchvision Resize(S): the short side becomes S, the long one int(S * long / short); CenterCrop: round-half-even offsets
    const int sh = min(d.h, d.w), lg = max(d.h, d.w);
    const int nl = (int)__ddiv_rn((double)((long long)S * lg), (double)sh);
    const int ow = d.w <= d.h ? S : nl, oh = d.w <= d.h ? nl : S;
    const int dy = oh - Ch, dx = ow - Cw;
    const int top = (dy >> 1) + ((dy & 1) & (dy >> 1)), left = (dx >> 1) + ((dx & 1) & (dx >> 1));
    if (tid < tw) win_h[tid] = et_window(et_pass(d.w, ow), left + ox0 + tid, kh[tid]);
    else if (tid >= ET_TW && tid - ET_TW < tr) win_v[tid - ET_TW] = et_window(et_pass(d.h, oh), top + oy0 + tid - ET_TW, kv[tid - ET_TW]);
  }
  __syncthreads();

  const int e = tid % ET_ELEMS, col = e / 3, c = e - 3 * col, half = tid / ET_ELEMS;
  int acc[ET_ROWS_PER_THREAD];
#pragma unroll
  for (int j = 0; j < ET_ROWS_PER_THREAD; ++j) acc[j] = 0;
  if (present) {
    const uint8_t* img = pixels + d.offset;
    const int y_lo = win_v[0].x, y_hi = win_v[tr - 1].x + win_v[tr - 1].y;   // windows move monotonically with the output row
    for (int y0 = y_lo; y0 < y_hi; y0 += ET_CHUNK) {
      const int nrows = min(ET_CHUNK, y_hi - y0);
      if (col < tw) {                                           // horizontal pass of chunk rows half, half + 2, ...
        const int2 wh = win_h[col];
        for (int r = half; r < nrows; r += 2) {
          const uint8_t* src = img + ((long long)(y0 + r) * d.w + wh.x) * 3 + c;
          int s = 1 << (ET_PRECISION_BITS - 1);
          for (int i = 0; i < wh.y; ++i) s += (int)__ldg(src + 3 * i) * kh[col][i];
          rows[r][e] = (uint8_t)et_clip8(s);
        }
      }
      __syncthreads();
#pragma unroll
      for (int j = 0; j < ET_ROWS_PER_THREAD; ++j) {            // vertical pass: this thread's rows whose windows meet the chunk
        const int oy = half * ET_ROWS_PER_THREAD + j;
        if (oy < tr) {
          const int2 wv = win_v[oy];
          const int ya = max(y0, wv.x), yb = min(y0 + nrows, wv.x + wv.y);
          for (int y = ya; y < yb; ++y) acc[j] += (int)rows[y - y0][e] * kv[oy][y - wv.x];
        }
      }
      __syncthreads();
    }
  }
  if (col < tw) {
#pragma unroll
    for (int j = 0; j < ET_ROWS_PER_THREAD; ++j) {
      const int oy = half * ET_ROWS_PER_THREAD + j;
      if (oy < tr) {
        const int u = present ? et_clip8(acc[j] + (1 << (ET_PRECISION_BITS - 1))) : 0;
        out[(((long long)b * Ch + oy0 + oy) * Cw + ox0 + col) * 3 + c] = lut[(c << 8) | u];
      }
    }
  }
}

}  // namespace hawq
