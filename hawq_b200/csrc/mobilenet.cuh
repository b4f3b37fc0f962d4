// MobileNetV2 layers the convolution kernel cannot run: the depthwise 3x3 convolutions (Q_LinearBottleneck.conv2 -> ReLU6 ->
// quant_act2) and the 3x3 stride-2 stem with 3 input channels (init_block -> ReLU6 -> quant_act_int32).  Both use conv_igemm's
// per-CTA channel set-up and requantisation policy (load_channel_block, with_rq, RqFp64 / RqExact), so they round exactly like
// its capped REQUANT epilogue, ReLU6 cap included (chan[c].reserved, folded into the upper clamp by load_channel_block).
#pragma once
#include "conv_igemm.cuh"

namespace hawq {

// ------------------------------------------------------------------------------------------------ depthwise 3x3
// 9 MACs per output: the layer is bound by memory traffic.  A thread owns 16 channels of one output column strip of DW_ROWS
// rows; a CTA is 256 neighbouring strips of the same 16 channels (one channel block, so the policy and the channel arrays are
// CTA-uniform and every shared-memory read is a broadcast).  Each input row is loaded once per strip with 16-byte vectors and kept
// in a rolling 3-row register window across the output rows that read it; the horizontally overlapping taps of neighbouring
// strips are served by L1.
constexpr int DW_CB = 16;     // channels per CTA (one 16-byte int8 vector per pixel)
constexpr int DW_ROWS = 8;    // output rows per strip
constexpr int DW_THREADS = 256;

// 16 channels c0 ... c0 + 15 of input pixel (n, hi, wi) as four int8x4 words; zeros outside the image.  A4: packed nibbles in
// hawq nibble order, expanded so that the words hold the same channels as in the 8-bit layout
template <bool A4>
__device__ __forceinline__ uint4 dw_load16(const ConvParams& p, int n, int hi, int wi, int c0) {
  if ((unsigned)hi >= (unsigned)p.H || (unsigned)wi >= (unsigned)p.W) return make_uint4(0u, 0u, 0u, 0u);
  const size_t e = ((size_t)(n * p.H + hi) * p.W + wi) * p.Cin + c0;
  if constexpr (A4) {
    const uint2 a = __ldg(reinterpret_cast<const uint2*>(p.x + (e >> 1)));
    return make_uint4(a.x & 0x0F0F0F0Fu, (a.x >> 4) & 0x0F0F0F0Fu, a.y & 0x0F0F0F0Fu, (a.y >> 4) & 0x0F0F0F0Fu);
  } else {
    return __ldg(reinterpret_cast<const uint4*>(p.x + e));
  }
}

// acc[j] += x[j] * w[j] for the 16 signed bytes of x and w
__device__ __forceinline__ void dw_mac16(int32_t (&acc)[16], const uint4& x, const uint4& w) {
  const uint32_t xs[4] = {x.x, x.y, x.z, x.w}, ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int b = 0; b < 4; ++b)
      acc[4 * k + b] += (int32_t)(int8_t)(xs[k] >> (8 * b)) * (int32_t)(int8_t)(ws[k] >> (8 * b));
}

// 16 requantised values -> 16 int8 bytes or 8 bytes of packed nibbles (hawq nibble order) at element offset e of dst
__device__ __forceinline__ void store_low16(void* dst, size_t e, const int32_t (&q)[16], int bits) {
  uint32_t wd[4];
#pragma unroll
  for (int k = 0; k < 4; ++k)
    wd[k] = __byte_perm(__byte_perm(q[4 * k], q[4 * k + 1], 0x0040), __byte_perm(q[4 * k + 2], q[4 * k + 3], 0x0040), 0x5410);
  uint8_t* o = reinterpret_cast<uint8_t*>(dst);
  if (bits == 8) *reinterpret_cast<uint4*>(o + e) = make_uint4(wd[0], wd[1], wd[2], wd[3]);
  else *reinterpret_cast<uint2*>(o + (e >> 1)) = make_uint2(pack_nibbles8(wd[0], wd[1]), pack_nibbles8(wd[2], wd[3]));
}

// p: N, H, W, Cin = Cout = C, stride, pad 1, Ho, Wo, w int8 [3][3][C], chan[C], relu, out_bits (8 / 4 packed), lo, hi.
template <bool A4>
__global__ void __launch_bounds__(DW_THREADS) dwconv3x3_kernel(const ConvParams p) {
  __shared__ __align__(16) uint8_t smem[ChanSmem<DW_CB>::BYTES];
  __shared__ uint4 sW[9];                                 // the CTA's 16 channels of the 9 taps (read as broadcasts)
  const ChanSmem<DW_CB> cs(smem);
  const int ncg = p.Cout / DW_CB;                         // channel groups fastest: the CTAs that read the same pixels run together
  const int c0 = (int)(blockIdx.x % ncg) * DW_CB;
  if (threadIdx.x < 9) sW[threadIdx.x] = __ldg(reinterpret_cast<const uint4*>(p.w + (size_t)threadIdx.x * p.Cout + c0));
  const RqPolicy pol = load_channel_block<DW_CB, false, true>(p, c0, cs);   // its barriers also publish sW

  const int spc = (p.Ho + DW_ROWS - 1) / DW_ROWS;       // strips per output column
  const long long s = (long long)(blockIdx.x / ncg) * DW_THREADS + threadIdx.x;
  if (s >= (long long)p.N * spc * p.Wo) return;           // ragged last CTA (no barrier follows)
  const int wo = (int)(s % p.Wo);
  const long long r = s / p.Wo;
  const int ho0 = (int)(r % spc) * DW_ROWS;
  const int n = (int)(r / spc);
  const int ho1 = min(ho0 + DW_ROWS, p.Ho);
  const int wi = wo * p.stride - 1;

  const int lo = p.relu ? min(max(p.lo, 0), p.hi) : p.lo;
  with_rq<false>(pol, p, [&](auto rq) {
    int hi = ho0 * p.stride - 1;                          // top input row of the window
    uint4 win[3][3];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) win[dy][dx] = dw_load16<A4>(p, n, hi + dy, wi + dx, c0);
    for (int ho = ho0;;) {
      int32_t acc[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[j] = 0;
#pragma unroll
      for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) dw_mac16(acc, win[dy][dx], sW[dy * 3 + dx]);
      int32_t q[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int4 c = *reinterpret_cast<const int4*>(&cs.chan[j]);   // bias, m, e, upper clamp
        q[j] = clampi(rq.term(rq.acc_bias(acc[j], cs.Cb[j], c.x), cs.M[j], c.y, c.z, false), lo, c.w);
      }
      store_low16(p.out, ((size_t)(n * p.Ho + ho) * p.Wo + wo) * p.Cout + c0, q, p.out_bits);
      if (++ho >= ho1) break;
      if (p.stride == 1) {                                // the window moves down one input row
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          win[0][dx] = win[1][dx];
          win[1][dx] = win[2][dx];
          win[2][dx] = dw_load16<A4>(p, n, hi + 3, wi + dx, c0);
        }
        hi += 1;
      } else {                                            // two input rows; the bottom row of the window becomes its top
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          win[0][dx] = win[2][dx];
          win[1][dx] = dw_load16<A4>(p, n, hi + 3, wi + dx, c0);
          win[2][dx] = dw_load16<A4>(p, n, hi + 4, wi + dx, c0);
        }
        hi += 2;
      }
    }
  });
}

// ------------------------------------------------------------------------------------------------ 3x3 stride-2 stem, Cin 3
// 27 MACs per output: CUDA cores suffice.  A pixel's 3 channels (+ a zero byte) are one 32-bit word, so each tap of each output
// channel is one dp4a.  A CTA computes STEM3_PX output pixels of one output row x 64 channels: warp w owns channels
// 16 * (w % 4) ... + 15 (warp-uniform: weight reads are broadcasts) of pixels 32 * (w / 4) + lane.  The 3 input rows it reads
// are staged in shared memory as one word per pixel.
constexpr int STEM3_PX = 64;
constexpr int STEM3_PW = 2 * STEM3_PX + 1;   // input columns of a CTA

// p: N, H, W, Ho, Wo, w int8 [64][3][3][4] (channel 3 zero), chan[64], relu, lo, hi, y_bits (16: int16, 32: int32) -> out,
// low_bits / low_m / low_e / low_lo / low_hi -> out_low (the next QuantAct's copy, scalar ratio).
__global__ void __launch_bounds__(256) stem3x3_kernel(const ConvParams p) {
  __shared__ __align__(16) uint8_t smem[ChanSmem<64>::BYTES];
  __shared__ uint32_t sW[9][64];
  __shared__ uint32_t sPatch[3][STEM3_PW];
  const ChanSmem<64> cs(smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tiles_x = (p.Wo + STEM3_PX - 1) / STEM3_PX;
  const int wo0 = (int)(blockIdx.x % tiles_x) * STEM3_PX;
  const long long r = blockIdx.x / tiles_x;
  const int ho = (int)(r % p.Ho), n = (int)(r / p.Ho);

  const uint32_t* w = reinterpret_cast<const uint32_t*>(p.w);
  for (int i = tid; i < 9 * 64; i += 256) sW[i % 9][i / 9] = w[i];
  for (int i = tid; i < 3 * STEM3_PW; i += 256) {
    const int dy = i / STEM3_PW, px = i - dy * STEM3_PW;
    const int iy = 2 * ho - 1 + dy, ix = 2 * wo0 - 1 + px;
    uint32_t v = 0;
    if ((unsigned)iy < (unsigned)p.H && (unsigned)ix < (unsigned)p.W) {
      const uint8_t* s = p.x + ((size_t)(n * p.H + iy) * p.W + ix) * 3;
      v = (uint32_t)s[0] | ((uint32_t)s[1] << 8) | ((uint32_t)s[2] << 16);
    }
    sPatch[dy][px] = v;
  }
  const RqPolicy pol = load_channel_block<64, false, true>(p, 0, cs);   // its barriers also publish sW and sPatch

  const int cb = (warp & 3) * 16;
  const int lx = (warp >> 2) * 32 + lane;
  const int wo = wo0 + lx;
  if (wo >= p.Wo) return;
  int32_t acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0;
#pragma unroll
  for (int dy = 0; dy < 3; ++dy)
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
      const int xw = (int)sPatch[dy][2 * lx + dx];
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[j] = __dp4a(xw, (int)sW[dy * 3 + dx][cb + j], acc[j]);
    }
  const size_t e = ((size_t)(n * p.Ho + ho) * p.Wo + wo) * 64 + cb;
  const int lo = p.relu ? min(max(p.lo, 0), p.hi) : p.lo;
  with_rq<false>(pol, p, [&](auto rq) {
    const double low_M = dyadic_to_double(p.low_m, p.low_e);
    int32_t q[16], ql[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int4 c = *reinterpret_cast<const int4*>(&cs.chan[cb + j]);   // bias, m, e, upper clamp
      q[j] = clampi(rq.term(rq.acc_bias(acc[j], cs.Cb[cb + j], c.x), cs.M[cb + j], c.y, c.z, false), lo, c.w);
      ql[j] = p.low_bits ? residual_low(rq, q[j], low_M, p) : 0;
    }
    if (p.y_bits == 16) {
      uint32_t h[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) h[k] = (uint32_t)(q[2 * k] & 0xFFFF) | ((uint32_t)q[2 * k + 1] << 16);
      int16_t* y = reinterpret_cast<int16_t*>(p.out) + e;
      *reinterpret_cast<uint4*>(y) = make_uint4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<uint4*>(y + 8) = make_uint4(h[4], h[5], h[6], h[7]);
    } else {
      int32_t* y = reinterpret_cast<int32_t*>(p.out) + e;
#pragma unroll
      for (int k = 0; k < 4; ++k) *reinterpret_cast<int4*>(y + 4 * k) = make_int4(q[4 * k], q[4 * k + 1], q[4 * k + 2], q[4 * k + 3]);
    }
    if (p.low_bits) store_low16(p.out_low, e, ql, p.low_bits);
  });
}

}  // namespace hawq
