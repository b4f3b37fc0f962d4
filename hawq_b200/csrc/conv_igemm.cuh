// Implicit-GEMM integer convolution with fused HAWQ epilogues (Hopper: warpgroup MMA + cp.async pipeline).
//
//   M = N*Ho*Wo output pixels, N = Cout, K = kh*kw*Cin.   A[m,k] gathered on the fly from the NHWC activation
//   tensor (zero-filled outside the image), B = int8 OHWI weights.  CTA tile 128 x BN x 64 channels, 2 warpgroups of
//   64 output rows each issuing wgmma m64nBNk32 (wgmma.cuh), 4-stage cp.async ring, shared-memory tiles in the
//   SWIZZLE_64B layout the wgmma descriptors read.
//
//   A4 = true: activations are packed unsigned nibbles (hawq nibble order).  They stay packed in HBM and in shared
//   memory (half the bytes); each ldmatrix word (8 nibbles) is expanded in registers with AND / SHIFT+AND into the
//   two int8x4 words of the register A fragment.  The weight rows of such layers are K-permuted on the host so that the
//   expansion needs no shuffles (hawq_permute_weights_for_i4).
//
//   DUAL = true (resize units): the identity-branch 1x1 convolution (x2, w2) runs first in the same CTA; its int32 result
//   (acc + bias2) stays in shared memory as the res_kind 1 operand of the RESIDUAL epilogue of the main convolution.
//
//   Epilogues (hawq_epilogue_mode): REQUANT (case 0 of fixedpoint_fn), RESIDUAL (case 1: dual dyadic requant + add,
//   optional ReLU, writes the new residual stream and/or the next unit's low-bit activation), RAW_I32, DEQUANT_F32.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"

namespace hawq {

struct ConvParams {
  const uint8_t* x;
  const int8_t* w;
  const hawq_chan* chan;
  const void* res;
  const hawq_chan* res_chan;
  const float* fscale;
  void* out;
  void* out_low;
  int32_t* status;
  int N, H, W, Cin, Cout, KH, KW, stride, pad, Ho, Wo, M, K;
  int cin_chunks;   // Cin / 64
  int x_pix_bytes;  // bytes per input pixel (Cin * a_bits / 8)
  int mode, relu, out_bits, lo, hi;
  int res_kind, res_bits;
  uint32_t res_m;
  int res_e;
  int y_bits, low_bits;
  uint32_t low_m;
  int low_e, low_lo, low_hi;
  int cout_store;
  int slow_scalar;   // host-checked: a scalar dyadic pair (res / low) has ratio > 1 -> generic 64-bit requant
  int wide_scalar_bad;   // host-checked: the scalar residual ratio exceeds 2^20 or the low-bit ratio exceeds 1 (no WIDE epilogue)
  int check_ovf;     // RESIDUAL under a HAWQ_EP_RATIOS_* promise: a requantised term leaving int32 raises HAWQ_FLAG_REQUANT_OVERFLOW
  int bias_lo, bias_hi;   // host-computed from K and a_bits: a bias in [bias_lo, bias_hi] keeps acc + bias inside int32 (empty when bias_lo > bias_hi)
  // DUAL launches: the identity 1x1 convolution (res_chan holds its bias and per-channel identity ratio)
  const uint8_t* x2;
  const int8_t* w2;
  int H2, W2, stride2, cin_chunks2, x2_pix_bytes;
};

constexpr int CONV_BM = 128;
constexpr int CONV_STAGES = 4;
constexpr int CONV_THREADS = 256;

// Shared memory of one CTA.  The cp.async ring is free once the GEMM has drained, so the epilogue tiles reuse it:
//   non-DUAL  [ ring | uint16 residual tile ] [ channel arrays ]
//             The uint16 residual tile has its own region: it is prefetched while the ring is in use (see gemm()).
//             After the GEMM the low-bit staging tile takes ring offset 0, and an int32 residual operand (loaded only after
//             the GEMM) starts right behind it, across the rest of the ring and the uint16 region.
//   DUAL      [ ring | int32 identity tile ] [ channel arrays ]
//             The identity tile is written after the identity GEMM and read by the main convolution's epilogue.  After the
//             main GEMM the low-bit tile (offset 0) and the uint16 stream tile (Y_OFF) are staged in the ring.
// Two CTAs per SM (what __launch_bounds__(CONV_THREADS, 2) plans for) need 2 * (TOTAL + 1 KB reserved per CTA) <= 228 KB.
template <int BN, bool A4, bool DUAL>
struct ConvSmem {
  static constexpr int A_ROW = A4 ? 32 : 64;  // bytes of one A row per k-tile (64 channels)
  static constexpr int A_STAGE = CONV_BM * A_ROW;
  static constexpr int B_STAGE = BN * 64;
  static constexpr int PIPE = CONV_STAGES * (A_STAGE + B_STAGE);
  static constexpr int OUT_PITCH = BN + 16;
  static constexpr int OUT_STAGE = CONV_BM * OUT_PITCH;                    // low-bit output staging tile, at offset 0
  static constexpr int RES16 = CONV_BM * (BN * 2 + 16);                    // uint16 tile (residual operand or stream), padded pitch
  static constexpr int RES32 = CONV_BM * (BN * 4 + 32);                    // int32 tile, padded pitch
  static constexpr int RES16_OFF = PIPE;
  static constexpr int RES32_OFF = DUAL ? PIPE : OUT_STAGE;
  static constexpr int Y_OFF = OUT_STAGE;                                  // DUAL: staged uint16 stream tile
  static constexpr int MAIN = DUAL ? PIPE + RES32 : (PIPE + RES16 > RES32_OFF + RES32 ? PIPE + RES16 : RES32_OFF + RES32);
  static constexpr int CHAN_OFF = MAIN;                                    // hawq_chan[BN]
  static constexpr int M_OFF = CHAN_OFF + BN * (int)sizeof(hawq_chan);     // double[BN]: m * 2^-e of chan
  static constexpr int M1_OFF = M_OFF + BN * 8;                           // double[BN]: m * 2^-e of res_chan
  static constexpr int RC_OFF = M1_OFF + BN * 8;                          // hawq_chan[BN]: res_chan
  static constexpr int CB_OFF = RC_OFF + BN * (int)sizeof(hawq_chan);     // double[BN]: 2^52 + 2^31 - bias
  static constexpr int TOTAL = CB_OFF + BN * 8;
  static_assert(OUT_STAGE <= PIPE && (!DUAL || Y_OFF + RES16 <= PIPE), "the epilogue staging tiles must fit in the freed ring");
  static_assert(2 * (TOTAL + 1024) <= 228 * 1024, "two CTAs per SM must fit in shared memory");
};

// swizzled byte offset of 16-byte chunk `ch` of row `row` (rows of 64 B: 4 chunks; rows of 32 B: 2 chunks)
template <int ROW_BYTES>
__device__ __forceinline__ int swz(int row, int ch) {
  if constexpr (ROW_BYTES == 64) return row * 64 + ((ch ^ ((row >> 1) & 3)) << 4);
  else return row * 32 + ((ch ^ ((row >> 2) & 1)) << 4);
}

// EPI selects the compile-time specialised fast epilogue (used when every dyadic ratio of the CTA is <= 1 and every bias keeps
// acc + bias inside int32, which the kernel verifies): 0 = none (generic run-time epilogue only), 1 = REQUANT to 4/8 bits, 2 = RESIDUAL.
constexpr int EPI_GENERIC = 0, EPI_FAST_LOW = 1, EPI_FAST_RES = 2;

// geometry of one implicit GEMM of a launch (the main convolution, or the identity convolution of a DUAL launch)
struct ConvGeom {
  const uint8_t* x;
  const int8_t* w;
  int H, W, stride, pad, KH, KW, cin_chunks, x_pix_bytes, K;
};

template <int BN, bool A4, int EPI, bool DUAL>
__global__ void __launch_bounds__(CONV_THREADS, 2) conv_igemm_kernel(const ConvParams p) {
  using S = ConvSmem<BN, A4, DUAL>;
  constexpr int BM = CONV_BM, STAGES = CONV_STAGES;
  constexpr int A_ROW = S::A_ROW;
  constexpr int A_CH = A_ROW / 16;                    // 16-byte chunks per A row: 4 or 2
  constexpr int A_ROWS_PER_PASS = CONV_THREADS / A_CH;  // 64 or 128
  constexpr int A_PASSES = BM / A_ROWS_PER_PASS;        // 2 or 1
  constexpr int B_PASSES = BN / 64;
  constexpr int NT = BN / 8;    // 8-column blocks of the accumulator: 16 or 8
  constexpr int NACC = BN / 2;  // accumulator registers per thread

  extern __shared__ __align__(1024) uint8_t smem[];   // 512-B aligned tiles: the wgmma descriptors address them swizzled
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * S::A_STAGE;
  hawq_chan* sChan = reinterpret_cast<hawq_chan*>(smem + S::CHAN_OFF);
  double* sM = reinterpret_cast<double*>(smem + S::M_OFF);
  double* sM1 = reinterpret_cast<double*>(smem + S::M1_OFF);
  hawq_chan* sResChan = reinterpret_cast<hawq_chan*>(smem + S::RC_OFF);
  double* sCb = reinterpret_cast<double*>(smem + S::CB_OFF);

  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int wg = warp >> 2;     // warpgroup: output rows 64 * wg ... 64 * wg + 63
  const int g = lane >> 2, t = lane & 3;
  // 1-D grid, row tile major: the Cout / BN CTAs that read the same 128 activation rows are launched back to back, so all but
  // the first find those rows in L2
  const int nblk = p.Cout / BN;
  const int m0 = (int)(blockIdx.x / nblk) * BM;
  const int n0 = (int)(blockIdx.x % nblk) * BN;

  int slow = p.slow_scalar;
  int wide_bad = p.wide_scalar_bad;   // some ratio > 2^20: the FP64 FMA is no longer exact for every int32 operand
  int bias_wide = 0;                  // some acc + bias may leave int32: the folded (unsaturated) bias add would differ from sat_add
  if (tid < BN) {
    const hawq_chan c = p.chan[n0 + tid];
    sChan[tid] = c;
    sM[tid] = dyadic_to_double(c.m, c.e);
    sCb[tid] = 4503601774854144.0 - (double)c.bias;   // exact: folds the bias add into the int -> double conversion
    bias_wide = c.bias < p.bias_lo || c.bias > p.bias_hi;
    slow |= !dyadic_is_fast(c.m, c.e);
    wide_bad |= !dyadic_is_wide(c.m, c.e);
    if (p.mode == HAWQ_EPI_RESIDUAL && p.res_kind == 1) {
      const hawq_chan rc = p.res_chan[n0 + tid];
      sResChan[tid] = rc;
      sM1[tid] = dyadic_to_double(rc.m, rc.e);
      slow |= !dyadic_is_fast(rc.m, rc.e);
      wide_bad |= !dyadic_is_wide(rc.m, rc.e);
    }
  }
  const bool use_slow = __syncthreads_or(slow) != 0;   // CTA-uniform: any ratio > 1 -> generic exact integer requant
  // RESIDUAL under a ratio promise with every ratio <= 2^20: the FP64 epilogue stays exact whenever a term fits int32, and every term
  // is range-checked (HAWQ_FLAG_REQUANT_OVERFLOW), so it replaces the generic epilogue (CTA-uniform)
  const bool use_wide = (__syncthreads_or(wide_bad) == 0) && use_slow && p.check_ovf && p.mode == HAWQ_EPI_RESIDUAL;
  // the specialised epilogues add the bias without saturating (sCb); a CTA with a bias near the int32 limits takes the
  // sat_add epilogue instead (CTA-uniform)
  const bool bias_fold = __syncthreads_or(bias_wide) == 0;

  int32_t acc[NACC];

  // RESIDUAL operand tile in shared memory; padded pitch keeps the fragment-pattern reads conflict-free
  const int res_es = (p.mode == HAWQ_EPI_RESIDUAL) ? ((p.res_kind == 1 || p.res_bits == 32) ? 4 : 2) : 0;
  const int res_pitch = BN * res_es + 8 * res_es;
  uint8_t* sRes = smem + (res_es == 2 ? S::RES16_OFF : S::RES32_OFF);

  // cp.async this CTA's tile of the residual operand into sRes (coalesced 16 B, zero-fill past M); no commit
  auto load_res = [&]() {
    const int cpr = BN * res_es / 16;   // 16-byte chunks per row
    const uint8_t* gres = reinterpret_cast<const uint8_t*>(p.res);
    for (int id = tid; id < BM * cpr; id += CONV_THREADS) {
      const int row = id / cpr, j = id - row * cpr;
      const bool v = m0 + row < p.M;
      const uint8_t* src = v ? gres + ((size_t)(m0 + row) * p.Cout + n0) * res_es + j * 16 : gres;
      cp_async_16(smem_u32(sRes + row * res_pitch + j * 16), src, v ? 16 : 0);
    }
  };
  // the uint16 residual operand has its own region: it is fetched while the GEMM runs (the int32 operand overlaps the ring)
  const bool prefetch_res = !DUAL && res_es == 2;

  // acc = A(128 x K) * B(K x BN) of geometry gm for this CTA's tile; with_res: the residual tile joins the prologue
  auto gemm = [&](const ConvGeom& gm, bool with_res) {
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0;
    // per-thread gather coordinates for the A rows this thread copies
    const int a_ch = tid % A_CH;
    int a_hi0[A_PASSES], a_wi0[A_PASSES], a_pix[A_PASSES];
    bool a_ok[A_PASSES];
#pragma unroll
    for (int i = 0; i < A_PASSES; ++i) {
      const int row = tid / A_CH + i * A_ROWS_PER_PASS;
      const int m = m0 + row;
      a_ok[i] = m < p.M;
      const int mm = a_ok[i] ? m : 0;
      const int n = mm / (p.Ho * p.Wo);
      const int r = mm - n * (p.Ho * p.Wo);
      const int ho = r / p.Wo, wo = r - ho * p.Wo;
      a_hi0[i] = ho * gm.stride - gm.pad;
      a_wi0[i] = wo * gm.stride - gm.pad;
      a_pix[i] = n * gm.H * gm.W;
    }
    const int b_ch = tid & 3, b_row = tid >> 2;
    const int KT = gm.KH * gm.KW * gm.cin_chunks;
    int ld_c = 0, ld_kw = 0, ld_kh = 0, ld_kt = 0;

    auto load_tile = [&](int stage) {
      const uint32_t a_base = smem_u32(sA + stage * S::A_STAGE);
#pragma unroll
      for (int i = 0; i < A_PASSES; ++i) {
        const int row = tid / A_CH + i * A_ROWS_PER_PASS;
        const int hi = a_hi0[i] + ld_kh, wi = a_wi0[i] + ld_kw;
        const bool v = a_ok[i] && (unsigned)hi < (unsigned)gm.H && (unsigned)wi < (unsigned)gm.W;
        const uint8_t* src = gm.x;
        if (v) src = gm.x + (size_t)(a_pix[i] + hi * gm.W + wi) * gm.x_pix_bytes + ld_c * A_ROW + a_ch * 16;
        cp_async_16(a_base + swz<A_ROW>(row, a_ch), src, v ? 16 : 0);
      }
      const uint32_t b_base = smem_u32(sB + stage * S::B_STAGE);
#pragma unroll
      for (int i = 0; i < B_PASSES; ++i) {
        const int row = b_row + i * 64;
        const int8_t* src = gm.w + (size_t)(n0 + row) * gm.K + ld_kt * 64 + b_ch * 16;
        cp_async_16(b_base + swz<64>(row, b_ch), src, 16);
      }
      ++ld_kt;
      if (++ld_c == gm.cin_chunks) {
        ld_c = 0;
        if (++ld_kw == gm.KW) { ld_kw = 0; ++ld_kh; }
      }
    };

    // cp.async groups retire in commit order.  The residual tile is issued right behind the prologue's k-tiles and
    // committed in their last group (k-tile STAGES - 2), so it is in flight during the whole GEMM: the waits for k-tiles
    // 0 ... STAGES - 3 never wait for it, and with KT < STAGES - 1 it is first waited for by the cp_async_wait<0> that
    // ends the GEMM.  Committed as a group of its own it would add one group to every later wait (each k-tile waited
    // for a stage early); committed first it would hold up k-tile 0.
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
      if (s < KT) load_tile(s);
      if (s == STAGES - 2 && with_res) load_res();
      cp_async_commit();
    }

    for (int kt = 0; kt < KT; ++kt) {
      cp_async_wait<STAGES - 2>();
      fence_proxy_async_smem();   // this thread's cp.async data -> visible to wgmma (async proxy)
      __syncthreads();            // every thread's data has landed; every warpgroup finished reading the stage refilled below
      if (kt + STAGES - 1 < KT) load_tile((kt + STAGES - 1) % STAGES);
      cp_async_commit();

      const int stage = kt % STAGES;
      const uint32_t a_base = smem_u32(sA + stage * S::A_STAGE);
      const uint32_t b_base = smem_u32(sB + stage * S::B_STAGE);
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {   // two k32 steps per 64-channel k-tile
        const uint64_t bdesc = wgmma_desc_sw64(b_base + ks * 32);
        if constexpr (!A4) {
          wgmma_fence();
          wgmma_ss<BN>(acc, wgmma_desc_sw64(a_base + wg * 64 * A_ROW + ks * 32), bdesc);
        } else {
          uint32_t r0, r1;
          const int row = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
          ldmatrix_x2(r0, r1, a_base + swz<32>(row, ks));
          const uint32_t af[4] = {r0 & 0x0F0F0F0Fu, r1 & 0x0F0F0F0Fu, (r0 >> 4) & 0x0F0F0F0Fu, (r1 >> 4) & 0x0F0F0F0Fu};
          wgmma_fence();
          wgmma_rs<BN>(acc, af, bdesc);
        }
      }
      wgmma_commit();
      wgmma_wait_all();
      fence_operands(acc);
    }
    cp_async_wait<0>();
    __syncthreads();   // pipeline buffers are free
  };

  if constexpr (DUAL) {   // identity convolution first: acc + bias2 (saturating) is the int32 res_kind 1 operand
    gemm(ConvGeom{p.x2, p.w2, p.H2, p.W2, p.stride2, 0, 1, 1, p.cin_chunks2, p.x2_pix_bytes, p.cin_chunks2 * 64}, false);
#pragma unroll
    for (int ni = 0; ni < NT; ++ni) {
      const int col = ni * 8 + 2 * t;
      const int b0 = sResChan[col].bias, b1 = sResChan[col + 1].bias;
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int row = warp * 16 + hf * 8 + g;
        *reinterpret_cast<int2*>(sRes + row * res_pitch + col * 4) =
            make_int2(sat_add(acc[ni * 4 + hf * 2], b0), sat_add(acc[ni * 4 + hf * 2 + 1], b1));
      }
    }
  }
  gemm(ConvGeom{p.x, p.w, p.H, p.W, p.stride, p.pad, p.KH, p.KW, p.cin_chunks, p.x_pix_bytes, p.K}, prefetch_res);

  if (!DUAL && res_es == 4) {   // int32 residual operand: its tile overlaps the ring, so it is loaded now
    load_res();
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
  }
  // the new residual stream is staged in shared memory and written with 16-byte stores: in place over the operand tile
  // when both have the same width, in the freed ring in DUAL launches (uint16 stream over an int32 identity tile)
  const bool y_staged = DUAL || (res_es != 0 && p.y_bits == res_es * 8);
  const int y_es = p.y_bits / 8;
  const int y_pitch = BN * y_es + 8 * y_es;
  uint8_t* sY = DUAL ? smem + S::Y_OFF : sRes;

  // ------------------------------------------------------------------------------------------------ epilogue
  uint8_t* sOut = smem;
  const bool stage_low = (p.mode == HAWQ_EPI_REQUANT && p.out_bits <= 8) || (p.mode == HAWQ_EPI_RESIDUAL && p.low_bits != 0);
  const int stage_bits = (p.mode == HAWQ_EPI_REQUANT) ? p.out_bits : p.low_bits;

  constexpr double kMagic = 6755399441055744.0;      // 1.5 * 2^52
  constexpr double kOffS = 4503601774854144.0;       // 2^52 + 2^31 (signed int -> double)
  constexpr double kOffU = 4503599627370496.0;       // 2^52        (non-negative int -> double)
  bool fast_done = false;

  if constexpr (EPI == EPI_FAST_LOW) {
    if (!use_slow && bias_fold) {
      fast_done = true;
      // clamp(RHE((acc + bias) * M)), ReLU folded into the lower clamp bound (RHE is monotone, RHE(0) = 0)
      const int lo = p.relu ? max(p.lo, 0) : p.lo, hi = p.hi;
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) {
        const int col = ni * 8 + 2 * t;
        const double2 Cb = *reinterpret_cast<const double2*>(&sCb[col]);
        const double2 M = *reinterpret_cast<const double2*>(&sM[col]);
        {
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            const int row = warp * 16 + hf * 8 + g;
            const double d0 = __hiloint2double(0x43300000, acc[ni * 4 + hf * 2 + 0] ^ 0x80000000) - Cb.x;
            const double d1 = __hiloint2double(0x43300000, acc[ni * 4 + hf * 2 + 1] ^ 0x80000000) - Cb.y;
            const int q0 = clampi(__double2loint(__fma_rn(d0, M.x, kMagic)), lo, hi);
            const int q1 = clampi(__double2loint(__fma_rn(d1, M.y, kMagic)), lo, hi);
            *reinterpret_cast<uint16_t*>(sOut + row * S::OUT_PITCH + col) = (uint16_t)__byte_perm(q0, q1, 0x0040);
          }
        }
      }
    }
  }

  if constexpr (EPI == EPI_FAST_RES) {
    if (bias_fold && (!use_slow || use_wide)) {
      fast_done = true;
      // t = fma(d, M, 1.5 * 2^52) with d * M exact inside the FMA: for |d * M| < 2^51 the low word of t is RHE(d * M); a term outside
      // int32 (which includes every |d * M| >= 2^51) is detected on t - 1.5 * 2^52 (exact in range, far out of range otherwise)
      bool ovf = false;
      auto term = [&](double d, double Mx, bool row_ok) -> int {
        const double tt = __fma_rn(d, Mx, kMagic);
        if (use_wide) {
          const double q = tt - kMagic;
          ovf |= row_ok && (q > 2147483647.0 || q < -2147483648.0);
        }
        return __double2loint(tt);
      };
      const double res_M = dyadic_to_double(p.res_m, p.res_e), low_M = dyadic_to_double(p.low_m, p.low_e);
      const int relu_floor = p.relu ? 0 : (int)0x80000000;
      int ymax = 0;
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) {
        const int col = ni * 8 + 2 * t;
        const double2 Cb = *reinterpret_cast<const double2*>(&sCb[col]);
        const double2 M = *reinterpret_cast<const double2*>(&sM[col]);
        double2 M1 = make_double2(res_M, res_M);
        if (p.res_kind == 1) M1 = *reinterpret_cast<const double2*>(&sM1[col]);
        {
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            const int row = warp * 16 + hf * 8 + g;
            const bool row_ok = m0 + row < p.M;
            const double d0 = __hiloint2double(0x43300000, acc[ni * 4 + hf * 2 + 0] ^ 0x80000000) - Cb.x;
            const double d1 = __hiloint2double(0x43300000, acc[ni * 4 + hf * 2 + 1] ^ 0x80000000) - Cb.y;
            const int v0 = term(d0, M.x, row_ok);
            const int v1 = term(d1, M.y, row_ok);
            uint8_t* rptr = sRes + row * res_pitch + col * res_es;
            double r0, r1;
            if (res_es == 2) {   // uint16 residual stream: non-negative, no sign fix-up
              const uint32_t pr = *reinterpret_cast<const uint32_t*>(rptr);
              r0 = __hiloint2double(0x43300000, (int)(pr & 0xFFFFu)) - kOffU;
              r1 = __hiloint2double(0x43300000, (int)(pr >> 16)) - kOffU;
            } else {
              const int2 pr = *reinterpret_cast<const int2*>(rptr);
              r0 = __hiloint2double(0x43300000, pr.x ^ 0x80000000) - kOffS;
              r1 = __hiloint2double(0x43300000, pr.y ^ 0x80000000) - kOffS;
            }
            int y0 = max(sat_add(term(r0, M1.x, row_ok), v0), relu_floor);
            int y1 = max(sat_add(term(r1, M1.y, row_ok), v1), relu_floor);
            uint8_t* yptr = sY + row * y_pitch + col * y_es;
            if (p.y_bits == 16) {
              if (row_ok) ymax = max(ymax, max(y0, y1));
              const uint32_t packed = (uint32_t)min(y0, 65535) | ((uint32_t)min(y1, 65535) << 16);
              if (y_staged) *reinterpret_cast<uint32_t*>(yptr) = packed;
              else if (m0 + row < p.M)
                *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out) + (size_t)(m0 + row) * p.Cout + n0 + col) = packed;
            } else if (p.y_bits == 32) {
              if (y_staged) *reinterpret_cast<int2*>(yptr) = make_int2(y0, y1);
              else if (m0 + row < p.M)
                *reinterpret_cast<int2*>(reinterpret_cast<int32_t*>(p.out) + (size_t)(m0 + row) * p.Cout + n0 + col) = make_int2(y0, y1);
            }
            if (p.low_bits != 0) {
              const double l0 = __hiloint2double(0x43300000, y0 ^ 0x80000000) - kOffS;
              const double l1 = __hiloint2double(0x43300000, y1 ^ 0x80000000) - kOffS;
              const int q0 = clampi(__double2loint(__fma_rn(l0, low_M, kMagic)), p.low_lo, p.low_hi);
              const int q1 = clampi(__double2loint(__fma_rn(l1, low_M, kMagic)), p.low_lo, p.low_hi);
              *reinterpret_cast<uint16_t*>(sOut + row * S::OUT_PITCH + col) = (uint16_t)__byte_perm(q0, q1, 0x0040);
            }
          }
        }
      }
      if (p.y_bits == 16 && ymax > 65535) atomicOr(p.status, HAWQ_FLAG_RESIDUAL_OVERFLOW);
      if (ovf) atomicOr(p.status, HAWQ_FLAG_REQUANT_OVERFLOW);
    }
  }

  auto epilogue = [&](auto fast_tag) {
    constexpr bool FAST = decltype(fast_tag)::value;
    const double res_M = dyadic_to_double(p.res_m, p.res_e), low_M = dyadic_to_double(p.low_m, p.low_e);
    auto rq = [&](int32_t v, uint32_t m, int e, double M) -> int32_t {
      if constexpr (FAST) return rhe_requant_fast(v, M);
      else return rhe_requant(v, m, e);
    };
    // the two terms of a RESIDUAL sum: under a ratio promise (check_ovf) a term outside int32 raises HAWQ_FLAG_REQUANT_OVERFLOW
    // (ratios <= 1, the FAST case, cannot leave int32)
    bool ovf = false;
    auto rq_term = [&](int32_t v, uint32_t m, int e, double M, bool row_ok) -> int32_t {
      if constexpr (FAST) {
        return rhe_requant_fast(v, M);
      } else {
        const long long q = rhe_requant64(v, m, e);
        ovf |= row_ok && (q > 2147483647ll || q < -2147483648ll);
        return sat_i32(q);
      }
    };
    {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int row = warp * 16 + hf * 8 + g;
        const int m = m0 + row;
        const bool ok = m < p.M;
#pragma unroll
        for (int ni = 0; ni < NT; ++ni) {
          const int col = ni * 8 + 2 * t;
          const int4 c0 = *reinterpret_cast<const int4*>(&sChan[col]);
          const int4 c1 = *reinterpret_cast<const int4*>(&sChan[col + 1]);
          const double2 M01 = *reinterpret_cast<const double2*>(&sM[col]);
          int32_t v0 = sat_add(acc[ni * 4 + hf * 2 + 0], c0.x);
          int32_t v1 = sat_add(acc[ni * 4 + hf * 2 + 1], c1.x);
          const size_t gidx = (size_t)m * p.Cout + n0 + col;
          if (p.mode == HAWQ_EPI_REQUANT) {
            if (p.relu) { v0 = max(v0, 0); v1 = max(v1, 0); }
            const int32_t q0 = clampi(rq(v0, (uint32_t)c0.y, c0.z, M01.x), p.lo, p.hi);
            const int32_t q1 = clampi(rq(v1, (uint32_t)c1.y, c1.z, M01.y), p.lo, p.hi);
            if (p.out_bits <= 8) {
              *reinterpret_cast<uint16_t*>(sOut + row * S::OUT_PITCH + col) = (uint16_t)((q0 & 0xFF) | ((q1 & 0xFF) << 8));
            } else if (ok) {
              if (p.out_bits == 16) {
                *reinterpret_cast<uint32_t*>(reinterpret_cast<int16_t*>(p.out) + gidx) =
                    (uint32_t)(q0 & 0xFFFF) | ((uint32_t)(q1 & 0xFFFF) << 16);
              } else {
                *reinterpret_cast<int2*>(reinterpret_cast<int32_t*>(p.out) + gidx) = make_int2(q0, q1);
              }
            }
          } else if (p.mode == HAWQ_EPI_RESIDUAL) {
            int32_t r0 = 0, r1 = 0;
            uint32_t rm0 = p.res_m, rm1 = p.res_m;
            int re0 = p.res_e, re1 = p.res_e;
            double rM0 = res_M, rM1 = res_M;
            uint8_t* rptr = sRes + row * res_pitch + col * res_es;
            if (res_es == 2) {
              const uint32_t pr = *reinterpret_cast<const uint32_t*>(rptr);
              r0 = (int32_t)(pr & 0xFFFFu);
              r1 = (int32_t)(pr >> 16);
            } else {
              const int2 pr = *reinterpret_cast<const int2*>(rptr);
              r0 = pr.x;
              r1 = pr.y;
            }
            if (p.res_kind == 1) {
              if constexpr (FAST) {
                const double2 M1 = *reinterpret_cast<const double2*>(&sM1[col]);
                rM0 = M1.x; rM1 = M1.y;
              } else {
                rm0 = sResChan[col].m; re0 = sResChan[col].e; rm1 = sResChan[col + 1].m; re1 = sResChan[col + 1].e;
              }
            }
            int32_t y0 = sat_add(rq_term(r0, rm0, re0, rM0, ok), rq_term(v0, (uint32_t)c0.y, c0.z, M01.x, ok));
            int32_t y1 = sat_add(rq_term(r1, rm1, re1, rM1, ok), rq_term(v1, (uint32_t)c1.y, c1.z, M01.y, ok));
            if (p.relu) { y0 = max(y0, 0); y1 = max(y1, 0); }
            uint8_t* yptr = sY + row * y_pitch + col * y_es;
            if (p.y_bits == 32) {
              if (y_staged) *reinterpret_cast<int2*>(yptr) = make_int2(y0, y1);
              else if (ok) *reinterpret_cast<int2*>(reinterpret_cast<int32_t*>(p.out) + gidx) = make_int2(y0, y1);
            } else if (p.y_bits == 16) {
              if (ok && max(y0, y1) > 65535) atomicOr(p.status, HAWQ_FLAG_RESIDUAL_OVERFLOW);
              const uint32_t packed = (uint32_t)min(y0, 65535) | ((uint32_t)min(y1, 65535) << 16);
              if (y_staged) *reinterpret_cast<uint32_t*>(yptr) = packed;
              else if (ok) *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out) + gidx) = packed;
            }
            if (p.low_bits != 0) {
              const int32_t q0 = clampi(rq(y0, p.low_m, p.low_e, low_M), p.low_lo, p.low_hi);
              const int32_t q1 = clampi(rq(y1, p.low_m, p.low_e, low_M), p.low_lo, p.low_hi);
              *reinterpret_cast<uint16_t*>(sOut + row * S::OUT_PITCH + col) = (uint16_t)((q0 & 0xFF) | ((q1 & 0xFF) << 8));
            }
          } else if (p.mode == HAWQ_EPI_RAW_I32) {
            if (ok) *reinterpret_cast<int2*>(reinterpret_cast<int32_t*>(p.out) + gidx) = make_int2(v0, v1);
          } else {  // HAWQ_EPI_DEQUANT_F32
            if (ok) {
              float* o = reinterpret_cast<float*>(p.out) + (size_t)m * p.cout_store;
              const int c = n0 + col;
              if (c < p.cout_store) o[c] = __fmul_rn((float)v0, p.fscale[c]);
              if (c + 1 < p.cout_store) o[c + 1] = __fmul_rn((float)v1, p.fscale[c + 1]);
            }
          }
        }
      }
    }
    if (ovf && p.check_ovf) atomicOr(p.status, HAWQ_FLAG_REQUANT_OVERFLOW);
  };
  if (!fast_done) {
    if (use_slow) epilogue(std::false_type{});
    else epilogue(std::true_type{});
  }

  if (y_staged || stage_low) __syncthreads();
  if (y_staged) {   // coalesced copy-out of the new residual stream tile
    const int cpr = BN * y_es / 16;
    uint8_t* gy = reinterpret_cast<uint8_t*>(p.out);
    for (int id = tid; id < BM * cpr; id += CONV_THREADS) {
      const int row = id / cpr, j = id - row * cpr;
      if (m0 + row < p.M)
        *reinterpret_cast<int4*>(gy + ((size_t)(m0 + row) * p.Cout + n0) * y_es + j * 16) =
            *reinterpret_cast<const int4*>(sY + row * y_pitch + j * 16);
    }
  }
  if (stage_low) {
    uint8_t* gout = reinterpret_cast<uint8_t*>(p.mode == HAWQ_EPI_REQUANT ? p.out : p.out_low);
    if (stage_bits == 8) {
      constexpr int CPR = BN / 16;
      for (int id = tid; id < BM * CPR; id += CONV_THREADS) {
        const int row = id / CPR, j = id % CPR;
        if (m0 + row < p.M) {
          const int4 v = *reinterpret_cast<const int4*>(sOut + row * S::OUT_PITCH + j * 16);
          *reinterpret_cast<int4*>(gout + (size_t)(m0 + row) * p.Cout + n0 + j * 16) = v;
        }
      }
    } else {  // 4-bit: 32 channels -> 16 packed bytes
      constexpr int CPR = BN / 32;
      for (int id = tid; id < BM * CPR; id += CONV_THREADS) {
        const int row = id / CPR, j = id % CPR;
        if (m0 + row < p.M) {
          const uint4 a = *reinterpret_cast<const uint4*>(sOut + row * S::OUT_PITCH + j * 32);
          const uint4 b = *reinterpret_cast<const uint4*>(sOut + row * S::OUT_PITCH + j * 32 + 16);
          uint4 o;
          o.x = pack_nibbles8(a.x, a.y);
          o.y = pack_nibbles8(a.z, a.w);
          o.z = pack_nibbles8(b.x, b.y);
          o.w = pack_nibbles8(b.z, b.w);
          *reinterpret_cast<uint4*>(gout + (((size_t)(m0 + row) * p.Cout + n0 + j * 32) >> 1)) = o;
        }
      }
    }
  }
}

}  // namespace hawq
