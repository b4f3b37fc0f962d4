// Persistent 1x1 convolution for the ResNet bottleneck tails (hawq_conv2d RESIDUAL, 1x1 stride 1, uint16 residual operand, uint16
// stream) and the resize units (hawq_conv2d_dual: a 1x1 main convolution plus a 1x1 identity convolution of stride 1 or 2).
//
//   These launches move many bytes per MAC (a stage-1 tail reads 64 activation bytes and 2 residual bytes per output channel row
//   and writes 3), so they are bound by HBM, not by the tensor cores.  Each CTA owns one channel block of BN columns for the
//   whole launch (its channel arrays and requantisation policy are set up once) and walks the row tiles rt0, rt0 + rstep, ...; the
//   CTAs that read the same 128 activation rows run side by side, so all but one find them in L2.
//
//   The cp.async ring of conv_igemm runs on across tile boundaries: the load counter continues into tile i + 1's k-tiles while tile
//   i's k-tiles are consumed, so tile i + 1's activations (and its uint16 residual tile, which has two slots) are in flight while tile
//   i's epilogue runs and its stores drain.  Every ring iteration commits exactly one cp.async group, so a wait for "all but the
//   last D - 1 groups" (D = prefetch distance in k-tiles) is a wait for the k-tile about to be consumed.  The residual tile of tile j
//   joins the group of j's first k-tile; it goes into slot j % 2, which tile j - 2 released before j - 1's first k-tile, as long as
//   D <= KT (one tile's k-tiles): D = min(STAGES - 1, KT) for the tails.
//
//   Resize units: the identity convolution's k-tiles come first in each tile; its requantised term RHE((acc2 + bias2) * ratio2)
//   (overflow check included) is the residual term of the main convolution's RESIDUAL epilogue.  Each thread parks its terms in
//   shared memory while the main GEMM runs and reads back only its own (as registers they would spill at two CTAs per SM), in a
//   [term pair][thread] layout: consecutive threads touch consecutive 8-byte words, free of bank conflicts.
//
//   The requantisation (RqFp64 / RqExact, residual_y, residual_low, stream16_pair, residual_flags) is conv_igemm.cuh's; the tile
//   loop is compiled once per implementation, chosen once per CTA.
#pragma once
#include "conv_igemm.cuh"

namespace hawq {

constexpr int TAIL_BN = 64;

// [ ring | resize units: int32 identity terms | uint16 tiles (two residual slots; resize units: one stream tile) | low-bit staging ]
// [ channel arrays ].  The new uint16 stream is staged in place over the residual tile it is computed from.
template <bool A4, bool DUAL>
struct TailSmem : ConvRing<TAIL_BN, A4> {
  using R = ConvRing<TAIL_BN, A4>;
  static constexpr int BN = TAIL_BN;
  static constexpr int Y_PITCH = tile_pitch(BN, 2);      // uint16 tile
  static constexpr int Y_SLOT = CONV_BM * Y_PITCH;
  static constexpr int I_OFF = R::PIPE;                  // identity terms: BN / 4 int2 per thread, [pair][thread]
  static constexpr int Y_OFF = I_OFF + (DUAL ? BN / 4 * CONV_THREADS * 8 : 0);
  static constexpr int Y_SLOTS = DUAL ? 1 : 2;
  static constexpr int OUT_OFF = Y_OFF + Y_SLOTS * Y_SLOT;
  static constexpr int CHAN_OFF = OUT_OFF + CONV_BM * R::OUT_PITCH;
  static constexpr int TOTAL = CHAN_OFF + ChanSmem<BN>::BYTES;
  static_assert(R::A_STAGE % 512 == 0 && R::B_STAGE % 512 == 0, "wgmma tiles must stay 512-B aligned");
  static_assert(Y_OFF % 16 == 0 && Y_SLOT % 16 == 0 && OUT_OFF % 16 == 0 && CHAN_OFF % 16 == 0, "16-byte copies need aligned tiles");
  static_assert(2 * (TOTAL + 1024) <= 228 * 1024, "two CTAs per SM must fit in shared memory");
};

// Grid of a tail launch: two CTAs per SM, rounded down to a multiple of the channel blocks (at least one of each).
inline int tail_grid(int Cout, int sm_count) {
  const int nblk = Cout / TAIL_BN;
  const int per = 2 * sm_count / nblk;
  return (per > 1 ? per : 1) * nblk;
}

template <bool A4, bool DUAL>
__global__ void __launch_bounds__(CONV_THREADS, 2) conv_tail_kernel(const ConvParams p) {
  using S = TailSmem<A4, DUAL>;
  constexpr int BN = TAIL_BN, BM = CONV_BM, STAGES = CONV_STAGES;
  constexpr int A_ROW = S::A_ROW, A_CH = S::A_CH, A_ROWS_PER_PASS = S::A_ROWS_PER_PASS, A_PASSES = S::A_PASSES;
  constexpr int NT = S::NT, NACC = S::NACC;

  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * S::A_STAGE;
  uint8_t* sOut = smem + S::OUT_OFF;
  const ChanSmem<BN> cs(smem + S::CHAN_OFF);

  const int tid = threadIdx.x;
  const AccFrag fr(tid);   // this thread's place in the accumulator layout

  const int nblk = p.Cout / BN;
  const int n0 = (int)(blockIdx.x % nblk) * BN;
  const int rt0 = (int)(blockIdx.x / nblk), rstep = (int)(gridDim.x / nblk);
  const int nrt = (p.M + BM - 1) / BM;
  if (rt0 >= nrt) return;                                  // CTA-uniform: no row tile for this CTA
  const int T = (nrt - rt0 + rstep - 1) / rstep;           // row tiles of this CTA

  const RqPolicy pol = load_channel_block<BN, true>(p, n0, cs);

  const int KT = p.cin_chunks;                             // main convolution k-tiles
  const int KT2 = DUAL ? p.cin_chunks2 : 0;                // identity convolution k-tiles (first in each tile)
  const int KTT = KT + KT2;
  const int D = DUAL ? STAGES - 1 : min(STAGES - 1, KT);   // prefetch distance in k-tiles

  // ---- loader: the next k-tile of the CTA's sequence (tile ld_t, k-tile ld_k); one commit per call, empty past the last tile
  int ld_t = 0, ld_k = 0, ld_s = 0;
  int ld_pix2[A_PASSES];   // resize units: identity input pixel of each A row this thread copies, set at the tile's first k-tile
  const int a_ch = tid % A_CH;
  const int b_ch = tid & 3, b_row = tid >> 2;
  auto issue = [&]() {
    if (ld_t < T) {
      const int lm0 = (rt0 + ld_t * rstep) * BM;
      const bool ident = DUAL && ld_k < KT2;
      const int kc = ident ? ld_k : ld_k - KT2;
      const uint8_t* xb = ident ? p.x2 : p.x;
      const int pix_bytes = ident ? p.x2_pix_bytes : p.x_pix_bytes;
      const uint32_t a_base = smem_u32(sA + ld_s * S::A_STAGE);
#pragma unroll
      for (int i = 0; i < A_PASSES; ++i) {
        const int row = tid / A_CH + i * A_ROWS_PER_PASS;
        const int m = lm0 + row;
        const bool v = m < p.M;
        if (DUAL && ld_k == 0 && v) {   // output pixel (n, ho, wo) reads identity input pixel (n, ho * stride2, wo * stride2)
          const int n = m / (p.Ho * p.Wo);
          const int r = m - n * (p.Ho * p.Wo);
          const int ho = r / p.Wo, wo = r - ho * p.Wo;
          ld_pix2[i] = (n * p.H2 + ho * p.stride2) * p.W2 + wo * p.stride2;
        }
        const uint8_t* src = xb;
        if (v) src = xb + (size_t)(ident ? ld_pix2[i] : m) * pix_bytes + kc * A_ROW + a_ch * 16;
        cp_async_16(a_base + swz<A_ROW>(row, a_ch), src, v ? 16 : 0);
      }
      const int8_t* wb = ident ? p.w2 : p.w;
      const int wk = (ident ? KT2 : KT) * 64;
      cp_async_16(smem_u32(sB + ld_s * S::B_STAGE) + swz<64>(b_row, b_ch), wb + (size_t)(n0 + b_row) * wk + kc * 64 + b_ch * 16, 16);
      // the tile's uint16 residual operand, into slot ld_t % 2.  Written out rather than through load_res_tile: with the shared
      // loader ptxas schedules this prologue differently and the stage-3 / 4 tails ran 0.5-1 % slower (H100 80GB HBM3, 700 W).
      if (!DUAL && ld_k == 0) {
        uint8_t* sr = smem + S::Y_OFF + (ld_t & 1) * S::Y_SLOT;
        const uint8_t* gres = reinterpret_cast<const uint8_t*>(p.res);
        constexpr int CPR = BN * 2 / 16;
        for (int id = tid; id < BM * CPR; id += CONV_THREADS) {
          const int row = id / CPR, j = id - row * CPR;
          const bool v = lm0 + row < p.M;
          const uint8_t* src = v ? gres + ((size_t)(lm0 + row) * p.Cout + n0) * 2 + j * 16 : gres;
          cp_async_16(smem_u32(sr + row * S::Y_PITCH + j * 16), src, v ? 16 : 0);
        }
      }
      if (++ld_k == KTT) { ld_k = 0; ++ld_t; }
      if (++ld_s == STAGES) ld_s = 0;
    }
    cp_async_commit();
  };

  int32_t acc[NACC];
  int cs_s = 0;   // ring stage of the next k-tile to consume
  // acc += the next k-tile of the sequence; refills the ring D k-tiles ahead
  auto consume = [&]() {
    if (D == 1) cp_async_wait<0>();
    else if (D == 2) cp_async_wait<1>();
    else cp_async_wait<2>();
    fence_proxy_async_smem();
    __syncthreads();   // every thread's data has landed; the stage refilled below and the tiles of the last epilogue are free
    issue();
    const uint32_t a_base = smem_u32(sA + cs_s * S::A_STAGE);
    const uint32_t b_base = smem_u32(sB + cs_s * S::B_STAGE);
    if (++cs_s == STAGES) cs_s = 0;
    mma_ktile<BN, A4>(acc, a_base, b_base);
  };

  for (int s = 0; s < D; ++s) issue();

  const double res_M = dyadic_to_double(p.res_m, p.res_e), low_M = dyadic_to_double(p.low_m, p.low_e);
  const int relu_floor = p.relu ? 0 : (int)0x80000000;
  uint8_t* gy = reinterpret_cast<uint8_t*>(p.out) + (size_t)n0 * 2;

  with_rq<true>(pol, p, [&](auto rq) {
    int ymax = 0;
    for (int j = 0; j < T; ++j) {
      const int m0 = (rt0 + j * rstep) * BM;
      if constexpr (DUAL) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = 0;
        for (int kt = 0; kt < KT2; ++kt) consume();
#pragma unroll
        for (int ni = 0; ni < NT; ++ni) {
          const int col = fr.col(ni);
          const int4 r0 = *reinterpret_cast<const int4*>(&cs.rc[col]);   // bias, m, e of the identity convolution
          const int4 r1 = *reinterpret_cast<const int4*>(&cs.rc[col + 1]);
          const double2 M1 = *reinterpret_cast<const double2*>(&cs.M1[col]);
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            const int row = fr.row(hf);
            const bool ok = m0 + row < p.M;
            const int i0 = acc_idx(ni, hf);
            *reinterpret_cast<int2*>(smem + S::I_OFF + ((ni * 2 + hf) * CONV_THREADS + tid) * 8) =
                make_int2(rq.term(rq.of_i32(sat_add(acc[i0], r0.x)), M1.x, r0.y, r0.z, ok),
                          rq.term(rq.of_i32(sat_add(acc[i0 + 1], r1.x)), M1.y, r1.y, r1.z, ok));
          }
        }
      }
#pragma unroll
      for (int i = 0; i < NACC; ++i) acc[i] = 0;
      for (int kt = 0; kt < KT; ++kt) consume();

      uint8_t* sY = smem + S::Y_OFF + (DUAL ? 0 : (j & 1) * S::Y_SLOT);
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) {
        const int col = fr.col(ni);
        const int4 c0 = *reinterpret_cast<const int4*>(&cs.chan[col]);   // bias, m, e
        const int4 c1 = *reinterpret_cast<const int4*>(&cs.chan[col + 1]);
        const double2 M = *reinterpret_cast<const double2*>(&cs.M[col]);
        const double2 Cb = *reinterpret_cast<const double2*>(&cs.Cb[col]);
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const int row = fr.row(hf);
          const bool ok = m0 + row < p.M;
          const int i0 = acc_idx(ni, hf);
          uint32_t* yp = reinterpret_cast<uint32_t*>(sY + row * S::Y_PITCH + col * 2);
          int32_t t0, t1;
          if constexpr (DUAL) {
            const int2 it = *reinterpret_cast<const int2*>(smem + S::I_OFF + ((ni * 2 + hf) * CONV_THREADS + tid) * 8);
            t0 = it.x;
            t1 = it.y;
          } else {
            const uint32_t pr = *yp;
            t0 = rq.term(rq.of_u16(pr & 0xFFFFu), res_M, p.res_m, p.res_e, ok);
            t1 = rq.term(rq.of_u16(pr >> 16), res_M, p.res_m, p.res_e, ok);
          }
          const int y0 = residual_y(rq, t0, acc[i0], Cb.x, c0, M.x, ok, relu_floor);
          const int y1 = residual_y(rq, t1, acc[i0 + 1], Cb.y, c1, M.y, ok, relu_floor);
          *yp = stream16_pair(y0, y1, ok, ymax);
          if (p.low_bits != 0) stage_low_pair(sOut, S::OUT_PITCH, row, col, residual_low(rq, y0, low_M, p), residual_low(rq, y1, low_M, p));
        }
      }
      __syncthreads();
      copy_out_rows(sY, S::Y_PITCH, gy, (size_t)p.Cout * 2, BN * 2, m0, p.M);
      if (p.low_bits != 0) copy_out_low<BN>(sOut, S::OUT_PITCH, reinterpret_cast<uint8_t*>(p.out_low), p.low_bits, m0, n0, p.M, p.Cout);
    }
    residual_flags(p, ymax, rq.ovf);
  });
  cp_async_wait<0>();   // the trailing groups are empty; nothing is left in flight at exit
}

}  // namespace hawq
