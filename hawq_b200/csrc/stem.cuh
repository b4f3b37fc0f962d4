// Stem of the quantized ResNets: 7x7 stride-2 pad-3 convolution with Cin = 3 (reference
// utils/models/q_resnet.py:117 quant_init_convbn) fused with bias, the 16-bit dyadic requant of quant_act_int32
// (q_resnet.py:120) and the ReLU (q_resnet.py:122).  Both commute with the 3x3 max-pool that sits between them in
// the reference (monotone, positive multiplier), so the pool runs afterwards on int16 (maxpool_requant_kernel).
//
// Direct convolution on tensor cores: a CTA owns an 8x16 tile of output pixels x all 64 channels.  The input patch
// (21 x 38 pixels) is staged in shared memory as one 32-bit word per pixel (3 channels + 0).  With the K order
// (kh, kw, c4) and kw padded 7 -> 8, one k32 MMA step is exactly one kernel row: the A fragment word of output
// pixel ox at tap kw is the patch word at column 2*ox + kw, i.e. plain LDS.32 with no im2col buffer.
//
// The channel set-up and the requantisation policy are conv_igemm's (load_channel_block, with_rq, RqFp64 / RqExact), so the stem
// rounds exactly like the convolution's REQUANT epilogue.
#pragma once
#include "conv_igemm.cuh"

namespace hawq {

constexpr int STEM_TH = 8, STEM_TW = 16;
constexpr int STEM_PH = 2 * STEM_TH + 5;  // 21
constexpr int STEM_PW = 2 * STEM_TW + 6;  // 38 (one extra column for the zero-weight 8th tap)
constexpr int STEM_WPITCH = 60;           // words per output channel in smem (7*8 = 56, padded: conflict-free)

// input patch of one 8x16 output tile (origin iy0, ix0 may lie outside the image: zero fill), one word per pixel; read-only loads
__device__ __forceinline__ void stem_load_patch(const uint8_t* x, int n, int H, int W, int iy0, int ix0, uint32_t* sPatch) {
  for (int i = threadIdx.x; i < STEM_PH * STEM_PW; i += 256) {
    const int py = i / STEM_PW, px = i - py * STEM_PW;
    const int iy = iy0 + py, ix = ix0 + px;
    uint32_t v = 0;
    if ((unsigned)iy < (unsigned)H && (unsigned)ix < (unsigned)W) {
      const uint8_t* s = x + ((size_t)(n * H + iy) * W + ix) * 3;
      v = (uint32_t)__ldg(s) | ((uint32_t)__ldg(s + 1) << 8) | ((uint32_t)__ldg(s + 2) << 16);
    }
    sPatch[i] = v;
  }
}

// raw accumulators of the 8x16 tile: warp w owns output row w; acc[j] = mma.m16n8 fragment of channels 8j..8j+7
// (fragment row g / g+8 = output column g / g+8)
__device__ __forceinline__ void stem_tile_mma(const uint32_t* sPatch, const uint32_t* sW, int32_t (&acc)[8][4]) {
  const int lane = threadIdx.x & 31, oy = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int k = 0; k < 4; ++k) acc[j][k] = 0;
#pragma unroll
  for (int kh = 0; kh < 7; ++kh) {
    const uint32_t* prow = sPatch + (2 * oy + kh) * STEM_PW;
    uint32_t a[4];
    a[0] = prow[2 * g + t];
    a[1] = prow[2 * (g + 8) + t];
    a[2] = prow[2 * g + 4 + t];
    a[3] = prow[2 * (g + 8) + 4 + t];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint32_t b[2];
      const uint32_t* wr = sW + (8 * j + g) * STEM_WPITCH + kh * 8;
      b[0] = wr[t];
      b[1] = wr[4 + t];
      mma_16832(acc[j], a, b);
    }
  }
}

// channels c, c + 1 of one convolution output: max(clamp(RHE((acc + bias) * ratio), lo, hi), 0) as an int16 pair.  The ReLU comes
// after the clamp (a negative clamp_hi gives 0), not folded into the lower bound as in conv_igemm's REQUANT.
template <class Rq>
__device__ __forceinline__ uint32_t stem_requant_pair(Rq& rq, const ChanSmem<64>& cs, int c, int32_t a0, int32_t a1, int lo, int hi) {
  const int4 c0 = *reinterpret_cast<const int4*>(&cs.chan[c]);   // bias, m, e
  const int4 c1 = *reinterpret_cast<const int4*>(&cs.chan[c + 1]);
  const int q0 = max(clampi(rq.term(rq.acc_bias(a0, cs.Cb[c], c0.x), cs.M[c], c0.y, c0.z, false), lo, hi), 0);
  const int q1 = max(clampi(rq.term(rq.acc_bias(a1, cs.Cb[c + 1], c1.x), cs.M[c + 1], c1.y, c1.z, false), lo, hi), 0);
  return (uint32_t)(q0 & 0xFFFF) | ((uint32_t)(q1 & 0xFFFF) << 16);
}

// Persistent: a grid of a few CTAs per SM loops over the 8x16 tiles (tile = (n, tile_y, tile_x) with x fastest), so the 14 KB of
// weights and the per-channel constants are staged once per CTA instead of once per tile (12 544 times per batch of 128).
// p: x, w (64 x 56 words), chan[64], N, H, W, Ho, Wo, lo, hi -> out (int16).
__global__ void __launch_bounds__(256) stem_conv_kernel(const ConvParams p) {
  __shared__ uint32_t sPatch[STEM_PH * STEM_PW];
  __shared__ uint32_t sW[64 * STEM_WPITCH];
  __shared__ __align__(16) uint8_t smem[ChanSmem<64>::BYTES];
  const ChanSmem<64> cs(smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(p.w);
  for (int i = tid; i < 64 * 56; i += 256) sW[(i / 56) * STEM_WPITCH + (i % 56)] = __ldg(w + i);
  const RqPolicy pol = load_channel_block<64, false>(p, 0, cs);   // its barriers also publish sW
  const int tiles_x = (p.Wo + STEM_TW - 1) / STEM_TW, tiles_y = (p.Ho + STEM_TH - 1) / STEM_TH;
  const long long total = (long long)p.N * tiles_y * tiles_x;
  for (long long tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const int tx = (int)(tile % tiles_x);
    const int ty = (int)((tile / tiles_x) % tiles_y);
    const int n = (int)(tile / ((long long)tiles_x * tiles_y));
    const int oy0 = ty * STEM_TH, ox0 = tx * STEM_TW;
    const int iy0 = oy0 * 2 - 3, ix0 = ox0 * 2 - 3;
    __syncthreads();                                   // the previous tile's patch has been consumed
    stem_load_patch(p.x, n, p.H, p.W, iy0, ix0, sPatch);
    __syncthreads();
    int32_t acc[8][4];
    stem_tile_mma(sPatch, sW, acc);
    const int oyg = oy0 + warp;                        // warp w owns output row w of the tile
    if (oyg >= p.Ho) continue;                         // (the barriers at the loop top are reached by every thread: no early exit)
    with_rq<false>(pol, p, [&](auto rq) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int oxg = ox0 + g + hf * 8;
        if (oxg >= p.Wo) continue;
        int16_t* o = reinterpret_cast<int16_t*>(p.out) + ((size_t)(n * p.Ho + oyg) * p.Wo + oxg) * 64;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = 8 * j + 2 * t;
          *reinterpret_cast<uint32_t*>(o + c) = stem_requant_pair(rq, cs, c, acc[j][hf * 2], acc[j][hf * 2 + 1], p.lo, p.hi);
        }
      }
    });
  }
}

// one pooled pixel x 8 channels (max of non-negative int16 values): residual stream y (uint16 / int32, 0 = none) and the
// first unit's quant_act output (case 0 with scalar m, e; int8 or packed nibbles, 0 = none)
__device__ __forceinline__ void pool_store(uint4 mx, size_t oidx, int y_bits, void* __restrict__ y, int low_bits, uint32_t low_m, int low_e,
                                           int low_lo, int low_hi, void* __restrict__ out_low) {
  int32_t v[8] = {(int)(mx.x & 0xFFFF), (int)(mx.x >> 16), (int)(mx.y & 0xFFFF), (int)(mx.y >> 16),
                  (int)(mx.z & 0xFFFF), (int)(mx.z >> 16), (int)(mx.w & 0xFFFF), (int)(mx.w >> 16)};
  if (y_bits == 16) {
    *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(y) + oidx) = mx;
  } else if (y_bits == 32) {
    int32_t* yo = reinterpret_cast<int32_t*>(y) + oidx;
    *reinterpret_cast<int4*>(yo) = make_int4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<int4*>(yo + 4) = make_int4(v[4], v[5], v[6], v[7]);
  }
  if (low_bits != 0) {
    uint32_t wlo = 0, whi = 0;
    const bool fast = dyadic_is_fast(low_m, low_e);
    const double low_M = dyadic_to_double(low_m, low_e);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int32_t qa = fast ? rhe_requant_fast(v[k], low_M) : rhe_requant(v[k], low_m, low_e);
      const int32_t qb = fast ? rhe_requant_fast(v[k + 4], low_M) : rhe_requant(v[k + 4], low_m, low_e);
      wlo |= (uint32_t)(clampi(qa, low_lo, low_hi) & 0xFF) << (8 * k);
      whi |= (uint32_t)(clampi(qb, low_lo, low_hi) & 0xFF) << (8 * k);
    }
    if (low_bits == 8) {
      *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(out_low) + oidx) = make_uint2(wlo, whi);
    } else {
      *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(out_low) + (oidx >> 1)) = pack_nibbles8(wlo, whi);
    }
  }
}

// nn.MaxPool2d(3, 2, 1) on the (non-negative) int16 stem output, then: residual stream y (uint16 / int32) and the
// first unit's quant_act output (case 0 with scalar m, e).  One thread = one output pixel x 8 channels.
__global__ void __launch_bounds__(256) maxpool_requant_kernel(const int16_t* __restrict__ x, int N, int H, int W, int C,
                                                              int Ho, int Wo, int y_bits, void* __restrict__ y,
                                                              int low_bits, uint32_t low_m, int low_e, int low_lo,
                                                              int low_hi, void* __restrict__ out_low) {
  const int c8 = C / 8;
  const long long total = (long long)N * Ho * Wo * c8;
  for (long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x; id < total;
       id += (long long)gridDim.x * blockDim.x) {
    const int cg = (int)(id % c8);
    long long r = id / c8;
    const int wo = (int)(r % Wo);
    r /= Wo;
    const int ho = (int)(r % Ho);
    const int n = (int)(r / Ho);
    uint4 mx = make_uint4(0, 0, 0, 0);  // inputs are >= 0, so 0 is a neutral padding value
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
      const int hi_ = ho * 2 - 1 + dy;
      if ((unsigned)hi_ >= (unsigned)H) continue;
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const int wi = wo * 2 - 1 + dx;
        if ((unsigned)wi >= (unsigned)W) continue;
        const uint4 v = *reinterpret_cast<const uint4*>(x + ((size_t)(n * H + hi_) * W + wi) * C + cg * 8);
        mx.x = __vmaxs2(mx.x, v.x);
        mx.y = __vmaxs2(mx.y, v.y);
        mx.z = __vmaxs2(mx.z, v.z);
        mx.w = __vmaxs2(mx.w, v.w);
      }
    }
    pool_store(mx, ((size_t)(n * Ho + ho) * Wo + wo) * C + cg * 8, y_bits, y, low_bits, low_m, low_e, low_lo, low_hi, out_low);
  }
}

// Fused stem (hawq_stem_pool_i8): convolution + bias + 16-bit requant + ReLU, max-pool 3x3/2, residual-stream store and low-bit
// copy in one kernel; the int16 convolution output only exists in shared memory.  Persistent CTAs loop over tiles of 3 x 7 pooled
// pixels, whose 3x3 windows cover the 7 x 15 convolution outputs starting at (2 * py0 - 1, 2 * px0 - 1): one 8x16 tile of the
// convolution above.  Positions outside the convolution output hold 0, neutral for the max of non-negative values.
constexpr int STEMP_PH = 3, STEMP_PW = 7;
// p: x, w (64 x 64 words, kernel rows 0..6 read), chan[64], N, H, W, Ho, Wo (convolution output), lo, hi, y_bits -> out,
// low_bits / low_m / low_e / low_lo / low_hi -> out_low.
__global__ void __launch_bounds__(256) stem_pool_kernel(const ConvParams p) {
  __shared__ uint32_t sPatch[STEM_PH * STEM_PW];
  __shared__ uint32_t sW[64 * STEM_WPITCH];
  __shared__ __align__(16) uint8_t smem[ChanSmem<64>::BYTES];
  __shared__ __align__(16) int16_t sConv[STEM_TH][STEM_TW][64];
  const ChanSmem<64> cs(smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const uint32_t* w256 = reinterpret_cast<const uint32_t*>(p.w);
  for (int i = tid; i < 64 * 56; i += 256) sW[(i / 56) * STEM_WPITCH + (i % 56)] = __ldg(w256 + (i / 56) * 64 + (i % 56));   // kernel rows 0..6
  const RqPolicy pol = load_channel_block<64, false>(p, 0, cs);   // its barriers also publish sW
  const int Po = (p.Ho - 1) / 2 + 1, Qo = (p.Wo - 1) / 2 + 1;      // max-pool 3x3 / 2, pad 1
  const int tiles_x = (Qo + STEMP_PW - 1) / STEMP_PW, tiles_y = (Po + STEMP_PH - 1) / STEMP_PH;
  const long long total = (long long)p.N * tiles_y * tiles_x;
  for (long long tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const int tx = (int)(tile % tiles_x);
    const int ty = (int)((tile / tiles_x) % tiles_y);
    const int n = (int)(tile / ((long long)tiles_x * tiles_y));
    const int py0 = ty * STEMP_PH, px0 = tx * STEMP_PW;
    const int oy0 = 2 * py0 - 1, ox0 = 2 * px0 - 1;
    __syncthreads();                                   // the previous tile's patch and convolution tile have been consumed
    stem_load_patch(p.x, n, p.H, p.W, oy0 * 2 - 3, ox0 * 2 - 3, sPatch);
    __syncthreads();
    int32_t acc[8][4];
    stem_tile_mma(sPatch, sW, acc);
    const int oyg = oy0 + warp;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int cx = g + hf * 8, oxg = ox0 + cx;
      const bool ok = (unsigned)oyg < (unsigned)p.Ho && (unsigned)oxg < (unsigned)p.Wo;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = 8 * j + 2 * t;
        // the policy is picked per pair: with one branch around the tile's 16 pairs ptxas interleaves them and this kernel needs
        // 118 registers instead of 56
        uint32_t q;
        with_rq<false>(pol, p, [&](auto rq) { q = stem_requant_pair(rq, cs, c, acc[j][hf * 2], acc[j][hf * 2 + 1], p.lo, p.hi); });
        *reinterpret_cast<uint32_t*>(&sConv[warp][cx][c]) = ok ? q : 0u;
      }
    }
    __syncthreads();
    for (int i = tid; i < STEMP_PH * STEMP_PW * 8; i += 256) {
      const int cg = i & 7, pix = i >> 3;
      const int ry = pix / STEMP_PW, rx = pix - ry * STEMP_PW;
      const int po = py0 + ry, qo = px0 + rx;
      if (po >= Po || qo >= Qo) continue;
      uint4 mx = make_uint4(0, 0, 0, 0);
#pragma unroll
      for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          const uint4 v = *reinterpret_cast<const uint4*>(&sConv[2 * ry + dy][2 * rx + dx][cg * 8]);
          mx.x = __vmaxs2(mx.x, v.x);
          mx.y = __vmaxs2(mx.y, v.y);
          mx.z = __vmaxs2(mx.z, v.z);
          mx.w = __vmaxs2(mx.w, v.w);
        }
      pool_store(mx, ((size_t)(n * Po + po) * Qo + qo) * 64 + cg * 8, p.y_bits, p.out, p.low_bits, p.low_m, p.low_e, p.low_lo, p.low_hi,
                 p.out_low);
    }
  }
}

}  // namespace hawq
