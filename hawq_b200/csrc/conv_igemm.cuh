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
//   Epilogues (hawq_epilogue_mode), one instantiation per family: REQUANT (case 0 of fixedpoint_fn), RESIDUAL (case 1: dual
//   dyadic requant + add, optional ReLU, writes the new residual stream and/or the next unit's low-bit activation), and STORE
//   (RAW_I32, DEQUANT_F32).  The REQUANT and RESIDUAL bodies are written once, over a requantisation implementation that each
//   CTA picks from its channels' ratios and biases (RqFp64: one FP64 FMA per term; RqExact: 64-bit integer arithmetic).
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
  int scalar_over_one;   // host-checked: a scalar dyadic pair (res / low) has ratio > 1
  int scalar_unchecked;  // host-checked: the scalar residual ratio exceeds 2^20 or the low-bit ratio exceeds 1 (no checked FP64 form)
  int check_ovf;     // RESIDUAL under a HAWQ_EP_RATIOS_* promise: a requantised term leaving int32 raises HAWQ_FLAG_REQUANT_OVERFLOW
  int bias_lo, bias_hi;   // host-computed from K and a_bits: a bias in [bias_lo, bias_hi] keeps acc + bias inside int32 (empty when bias_lo > bias_hi)
  // resize units (conv_tail.cuh): the identity 1x1 convolution (res_chan holds its bias and per-channel identity ratio)
  const uint8_t* x2;
  const int8_t* w2;
  int H2, W2, stride2, cin_chunks2, x2_pix_bytes;
};

constexpr int CONV_BM = 128;
constexpr int CONV_STAGES = 4;
constexpr int CONV_THREADS = 256;

// Per-channel arrays of a CTA's channel block (BN channels), behind the tiles of its shared memory.
template <int BN>
struct ChanSmem {
  static constexpr int M_OFF = BN * (int)sizeof(hawq_chan);    // double[BN]: m * 2^-e of chan
  static constexpr int M1_OFF = M_OFF + BN * 8;                // double[BN]: m * 2^-e of res_chan
  static constexpr int RC_OFF = M1_OFF + BN * 8;               // hawq_chan[BN]: res_chan
  static constexpr int CB_OFF = RC_OFF + BN * (int)sizeof(hawq_chan);   // double[BN]: 2^52 + 2^31 - bias
  static constexpr int BYTES = CB_OFF + BN * 8;
  hawq_chan* chan;
  double* M;
  double* M1;
  hawq_chan* rc;
  double* Cb;
  __device__ explicit ChanSmem(uint8_t* base)
      : chan(reinterpret_cast<hawq_chan*>(base)), M(reinterpret_cast<double*>(base + M_OFF)),
        M1(reinterpret_cast<double*>(base + M1_OFF)), rc(reinterpret_cast<hawq_chan*>(base + RC_OFF)),
        Cb(reinterpret_cast<double*>(base + CB_OFF)) {}
};

// The cp.async ring of the convolution kernels (conv_igemm_kernel, conv_tail_kernel): CONV_STAGES stages of a 128-row A tile and a
// BN-row B tile of one 64-channel k-tile, at the front of shared memory; the per-thread A copy passes and accumulator count.
template <int BN, bool A4>
struct ConvRing {
  static constexpr int A_ROW = A4 ? 32 : 64;                    // bytes of one A row per k-tile (64 channels)
  static constexpr int A_STAGE = CONV_BM * A_ROW;
  static constexpr int B_STAGE = BN * 64;
  static constexpr int PIPE = CONV_STAGES * (A_STAGE + B_STAGE);
  static constexpr int A_CH = A_ROW / 16;                       // 16-byte chunks per A row: 4 or 2
  static constexpr int A_ROWS_PER_PASS = CONV_THREADS / A_CH;   // 64 or 128
  static constexpr int A_PASSES = CONV_BM / A_ROWS_PER_PASS;    // 2 or 1
  static constexpr int NT = BN / 8;                             // 8-column blocks of the accumulator: 16 or 8
  static constexpr int NACC = BN / 2;                           // accumulator registers per thread
  static constexpr int OUT_PITCH = BN + 16;                     // low-bit staging tile, one byte per value
};

// pitch of a shared-memory tile of BN es-byte elements per row (residual operand, new stream): 8 elements of padding keep the
// fragment-pattern reads conflict-free
__host__ __device__ constexpr int tile_pitch(int bn, int es) { return (bn + 8) * es; }

// Shared memory of one CTA.  The cp.async ring is free once the GEMM has drained, so the epilogue tiles reuse it:
//   [ ring | uint16 residual tile ] [ channel arrays ]
//   The uint16 residual tile has its own region: it is prefetched while the ring is in use (see gemm()).  After the GEMM the
//   low-bit staging tile takes ring offset 0, and an int32 residual operand (loaded only after the GEMM) starts right behind it,
//   across the rest of the ring and the uint16 region.
// Two CTAs per SM (what __launch_bounds__(CONV_THREADS, 2) plans for) need 2 * (TOTAL + 1 KB reserved per CTA) <= 228 KB.
template <int BN, bool A4>
struct ConvSmem : ConvRing<BN, A4> {
  using R = ConvRing<BN, A4>;
  static constexpr int OUT_STAGE = CONV_BM * R::OUT_PITCH;                 // low-bit output staging tile, at offset 0
  static constexpr int RES16 = CONV_BM * tile_pitch(BN, 2);                // uint16 residual tile
  static constexpr int RES32 = CONV_BM * tile_pitch(BN, 4);                // int32 tile
  static constexpr int RES16_OFF = R::PIPE;
  static constexpr int RES32_OFF = OUT_STAGE;
  static constexpr int MAIN = R::PIPE + RES16 > RES32_OFF + RES32 ? R::PIPE + RES16 : RES32_OFF + RES32;
  static constexpr int CHAN_OFF = MAIN;
  static constexpr int TOTAL = CHAN_OFF + ChanSmem<BN>::BYTES;
  static_assert(OUT_STAGE <= R::PIPE, "the low-bit staging tile must fit in the freed ring");
  static_assert(2 * (TOTAL + 1024) <= 228 * 1024, "two CTAs per SM must fit in shared memory");
};

// swizzled byte offset of 16-byte chunk `ch` of row `row` (rows of 64 B: 4 chunks; rows of 32 B: 2 chunks)
template <int ROW_BYTES>
__device__ __forceinline__ int swz(int row, int ch) {
  if constexpr (ROW_BYTES == 64) return row * 64 + ((ch ^ ((row >> 1) & 3)) << 4);
  else return row * 32 + ((ch ^ ((row >> 2) & 1)) << 4);
}

// acc += one 64-channel k-tile of the ring stage at a_base / b_base (shared-memory addresses): two k32 wgmma steps of the thread's
// warpgroup, waited for.  A4: each ldmatrix word (8 packed nibbles) is expanded with AND / SHIFT+AND into the two int8x4 words of
// the register A fragment.
template <int BN, bool A4>
__device__ __forceinline__ void mma_ktile(int32_t (&acc)[BN / 2], uint32_t a_base, uint32_t b_base) {
  constexpr int A_ROW = ConvRing<BN, A4>::A_ROW;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    const uint64_t bdesc = wgmma_desc_sw64(b_base + ks * 32);
    if constexpr (!A4) {
      wgmma_fence();
      wgmma_ss<BN>(acc, wgmma_desc_sw64(a_base + (warp >> 2) * 64 * A_ROW + ks * 32), bdesc);
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

// cp.asyncs rows m0 ... m0 + CONV_BM - 1, columns n0 ... n0 + BN - 1 of the residual operand p.res (es-byte elements, Cout per row)
// into the shared-memory tile s of pitch tile_pitch(BN, es): coalesced 16-byte copies, zero-filled past M; no commit
template <int BN>
__device__ __forceinline__ void load_res_tile(uint8_t* s, const ConvParams& p, int es, int m0, int n0) {
  const int cpr = BN * es / 16;   // 16-byte chunks per row
  const uint8_t* g = reinterpret_cast<const uint8_t*>(p.res);
  for (int id = threadIdx.x; id < CONV_BM * cpr; id += CONV_THREADS) {
    const int row = id / cpr, j = id - row * cpr;
    const bool v = m0 + row < p.M;
    const uint8_t* src = v ? g + ((size_t)(m0 + row) * p.Cout + n0) * es + j * 16 : g;
    cp_async_16(smem_u32(s + row * tile_pitch(BN, es) + j * 16), src, v ? 16 : 0);
  }
}

// Epilogue family of an instantiation (FAM): REQUANT to 4/8/16/32 bits, RESIDUAL, STORE (RAW_I32 and
// DEQUANT_F32, no requantisation), and REQUANT with per-channel ReLU6 caps (relu 2).  A kernel carries its own family's body only;
// the capped REQUANT has its own copy so that the uncapped one (relu 0 / 1) keeps its code and registers.
constexpr int FAM_REQUANT = 0, FAM_RESIDUAL = 1, FAM_STORE = 2, FAM_REQUANT_CAPPED = 3;

// One requantised term q = RHE(value * m / 2^e) of an epilogue, in one of two implementations; the kernel picks one per CTA.
// Operands are built by acc_bias (acc + bias of a channel), of_i32 and of_u16; term() takes the ratio both as M = m * 2^-e and as
// (m, e), and with `count` set a result outside int32 raises HAWQ_FLAG_REQUANT_OVERFLOW when the CTA is `checked`.
//
// FP64: an operand is its value as an exact double, built from bits without a conversion instruction ({0x43300000, v ^ 0x80000000}
// is 2^52 + 2^31 + v; the channel's sCb = 2^52 + 2^31 - bias folds the bias add into it).  t = fma(d, M, 1.5 * 2^52) rounds the
// exact product once, ties to even, and its low word is q whenever |d * M| < 2^51: always for ratios <= 1 (|q| <= |d| <= 2^31).
// For ratios up to 2^20 (checked) d * M is still exact inside the FMA and t - 1.5 * 2^52 is exact while q fits int32 and far outside
// int32 otherwise, so one compare pair detects every overflow.  CLAMPED: some bias of the CTA can take acc + bias out of int32, so
// that sum is clamped to int32 (d is exact, so the clamp equals sat_add); a compile-time flag keeps the clamp off the common path.
template <bool CLAMPED>
struct RqFp64 {
  bool checked;
  bool ovf = false;
  static constexpr double kMagic = 6755399441055744.0;   // 1.5 * 2^52
  __device__ static double acc_bias(int32_t acc, double cb, int32_t) {
    const double d = __hiloint2double(0x43300000, acc ^ 0x80000000) - cb;
    return CLAMPED ? fmin(fmax(d, -2147483648.0), 2147483647.0) : d;
  }
  __device__ static double of_i32(int32_t v) {
    return __hiloint2double(0x43300000, v ^ 0x80000000) - 4503601774854144.0;   // - (2^52 + 2^31)
  }
  __device__ static double of_u16(uint32_t u) { return __hiloint2double(0x43300000, (int)u) - 4503599627370496.0; }   // - 2^52
  __device__ int32_t term(double d, double M, uint32_t, int32_t, bool count) {
    const double t = __fma_rn(d, M, kMagic);
    if (checked && count) {
      const double q = t - kMagic;
      ovf |= q > 2147483647.0 || q < -2147483648.0;
    }
    return __double2loint(t);
  }
};
// Exact: rhe_requant64 of the saturated int32 value, for any ratio, saturated to int32.
struct RqExact {
  bool checked;
  bool ovf = false;
  __device__ static int32_t acc_bias(int32_t acc, double, int32_t bias) { return sat_add(acc, bias); }
  __device__ static int32_t of_i32(int32_t v) { return v; }
  __device__ static int32_t of_u16(uint32_t u) { return (int32_t)u; }
  __device__ int32_t term(int32_t v, double, uint32_t m, int32_t e, bool count) {
    const long long q = rhe_requant64(v, m, e);
    if (checked && count) ovf |= q > 2147483647ll || q < -2147483648ll;
    return sat_i32(q);
  }
};

// Requantisation policy of a CTA, from its channel block and the launch's scalar ratios: FP64 when every ratio is <= 1, and for
// RESIDUAL under a ratio promise when every ratio is <= 2^20 (the low-bit ratio <= 1), each term then checked; Exact otherwise.
// An FP64 CTA with a bias outside the window clamps.
struct RqPolicy {
  bool over_one;    // some ratio > 1
  bool unchecked;   // some ratio > 2^20 (or a low-bit ratio > 1): beyond the checked FP64 form
  bool clamped;     // some bias outside [bias_lo, bias_hi]: acc + bias may leave int32
};

// Loads the channel block n0 ... n0 + BN - 1 (and, for a res_kind 1 RESIDUAL, its res_chan) into shared memory and returns the
// CTA's policy.  CAPS: .reserved becomes the channel's upper clamp, min(hi, reserved) under relu 2 (ReLU6), else hi.  Every thread
// of the CTA must call it (three __syncthreads_or).
template <int BN, bool RESIDUAL, bool CAPS = false>
__device__ RqPolicy load_channel_block(const ConvParams& p, int n0, const ChanSmem<BN>& cs) {
  int over_one = p.scalar_over_one, unchecked = p.scalar_unchecked, bias_out = 0;
  const int tid = threadIdx.x;
  if (tid < BN) {
    hawq_chan c = p.chan[n0 + tid];
    if (CAPS) c.reserved = p.relu == 2 ? min(p.hi, c.reserved) : p.hi;
    cs.chan[tid] = c;
    cs.M[tid] = dyadic_to_double(c.m, c.e);
    cs.Cb[tid] = 4503601774854144.0 - (double)c.bias;   // exact: folds the bias add into the int -> double conversion
    bias_out = c.bias < p.bias_lo || c.bias > p.bias_hi;
    over_one |= !dyadic_is_fast(c.m, c.e);
    unchecked |= !dyadic_is_wide(c.m, c.e);
    if (RESIDUAL && p.res_kind == 1) {
      const hawq_chan rc = p.res_chan[n0 + tid];
      cs.rc[tid] = rc;
      cs.M1[tid] = dyadic_to_double(rc.m, rc.e);
      over_one |= !dyadic_is_fast(rc.m, rc.e);
      unchecked |= !dyadic_is_wide(rc.m, rc.e);
    }
  }
  RqPolicy pol;
  pol.over_one = __syncthreads_or(over_one) != 0;
  pol.unchecked = __syncthreads_or(unchecked) != 0;
  pol.clamped = __syncthreads_or(bias_out) != 0;
  return pol;
}

// Calls f with the requantisation implementation of the policy (RqExact, RqFp64<true> or RqFp64<false>), checked as RESIDUAL needs.
template <bool RESIDUAL, class F>
__device__ __forceinline__ void with_rq(const RqPolicy& pol, const ConvParams& p, F&& f) {
  const bool fp64 = !pol.over_one || (RESIDUAL && p.check_ovf && !pol.unchecked);
  if (!fp64) f(RqExact{RESIDUAL && p.check_ovf != 0});
  else if (pol.clamped) f(RqFp64<true>{RESIDUAL && pol.over_one});
  else f(RqFp64<false>{RESIDUAL && pol.over_one});
}

// RESIDUAL epilogue of one output: y = [ReLU](sat_add(res_term, RHE((acc + bias) * ratio))), where res_term = RHE(r * ratio1) of
// the residual operand r; with `ok` (a real row) a term leaving int32 counts for HAWQ_FLAG_REQUANT_OVERFLOW.
template <class Rq>
__device__ __forceinline__ int32_t residual_y(Rq& rq, int32_t res_term, int32_t acc, double cb, const int4& c, double M, bool ok,
                                              int32_t relu_floor) {
  return max(sat_add(res_term, rq.term(rq.acc_bias(acc, cb, c.x), M, c.y, c.z, ok)), relu_floor);
}
// the low-bit copy of y for the next unit: clamp(RHE(y * low ratio))
template <class Rq>
__device__ __forceinline__ int32_t residual_low(Rq& rq, int32_t y, double low_M, const ConvParams& p) {
  return clampi(rq.term(rq.of_i32(y), low_M, p.low_m, p.low_e, false), p.low_lo, p.low_hi);
}
// a pair of the uint16 stream: saturates at 65535; ymax keeps the largest value of real rows for HAWQ_FLAG_RESIDUAL_OVERFLOW
__device__ __forceinline__ uint32_t stream16_pair(int32_t y0, int32_t y1, bool ok, int& ymax) {
  if (ok) ymax = max(ymax, max(y0, y1));
  return (uint32_t)min(y0, 65535) | ((uint32_t)min(y1, 65535) << 16);
}
__device__ __forceinline__ void residual_flags(const ConvParams& p, int ymax, bool ovf) {
  if (ymax > 65535) atomicOr(p.status, HAWQ_FLAG_RESIDUAL_OVERFLOW);
  if (ovf) atomicOr(p.status, HAWQ_FLAG_REQUANT_OVERFLOW);
}
// a pair of low-bit outputs (columns col, col + 1) into a staging tile of one byte per value
__device__ __forceinline__ void stage_low_pair(uint8_t* s, int pitch, int row, int col, int q0, int q1) {
  *reinterpret_cast<uint16_t*>(s + row * pitch + col) = (uint16_t)__byte_perm(q0, q1, 0x0040);
}

// Coalesced 16-byte copy-out of a staged tile of CONV_BM rows: row r (row_bytes at s + r * s_pitch) goes to g + (m0 + r) * g_pitch;
// rows at or past M are skipped.  The caller synchronises before.
__device__ __forceinline__ void copy_out_rows(const uint8_t* s, int s_pitch, uint8_t* g, size_t g_pitch, int row_bytes, int m0, int M) {
  const int cpr = row_bytes / 16;
  for (int id = threadIdx.x; id < CONV_BM * cpr; id += blockDim.x) {
    const int row = id / cpr, j = id - row * cpr;
    if (m0 + row < M)
      *reinterpret_cast<int4*>(g + (size_t)(m0 + row) * g_pitch + j * 16) = *reinterpret_cast<const int4*>(s + row * s_pitch + j * 16);
  }
}
// The low-bit staging tile (one byte per value, BN columns) -> 8-bit rows, or 4-bit rows packed in hawq nibble order.
template <int BN>
__device__ __forceinline__ void copy_out_low(const uint8_t* s, int pitch, uint8_t* gout, int bits, int m0, int n0, int M, int Cout) {
  if (bits == 8) {
    copy_out_rows(s, pitch, gout + n0, (size_t)Cout, BN, m0, M);
  } else {  // 32 channels -> 16 packed bytes
    constexpr int CPR = BN / 32;
    for (int id = threadIdx.x; id < CONV_BM * CPR; id += blockDim.x) {
      const int row = id / CPR, j = id % CPR;
      if (m0 + row < M) {
        const uint4 a = *reinterpret_cast<const uint4*>(s + row * pitch + j * 32);
        const uint4 b = *reinterpret_cast<const uint4*>(s + row * pitch + j * 32 + 16);
        uint4 o;
        o.x = pack_nibbles8(a.x, a.y);
        o.y = pack_nibbles8(a.z, a.w);
        o.z = pack_nibbles8(b.x, b.y);
        o.w = pack_nibbles8(b.z, b.w);
        *reinterpret_cast<uint4*>(gout + (((size_t)(m0 + row) * Cout + n0 + j * 32) >> 1)) = o;
      }
    }
  }
}

// geometry of the implicit GEMM of a launch
struct ConvGeom {
  const uint8_t* x;
  const int8_t* w;
  int H, W, stride, pad, KH, KW, cin_chunks, x_pix_bytes, K;
};

template <int BN, bool A4, int FAM>
__global__ void __launch_bounds__(CONV_THREADS, 2) conv_igemm_kernel(const ConvParams p) {
  using S = ConvSmem<BN, A4>;
  constexpr int BM = CONV_BM, STAGES = CONV_STAGES;
  constexpr int A_ROW = S::A_ROW, A_CH = S::A_CH, A_ROWS_PER_PASS = S::A_ROWS_PER_PASS, A_PASSES = S::A_PASSES;
  constexpr int NT = S::NT, NACC = S::NACC;
  constexpr int B_PASSES = BN / 64;

  extern __shared__ __align__(1024) uint8_t smem[];   // 512-B aligned tiles: the wgmma descriptors address them swizzled
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * S::A_STAGE;
  const ChanSmem<BN> cs(smem + S::CHAN_OFF);
  const hawq_chan* sChan = cs.chan;
  const double* sM = cs.M;
  const double* sM1 = cs.M1;
  const hawq_chan* sResChan = cs.rc;
  const double* sCb = cs.Cb;

  const int tid = threadIdx.x;
  const AccFrag fr(tid);   // this thread's place in the accumulator layout
  // 1-D grid, row tile major: the Cout / BN CTAs that read the same 128 activation rows are launched back to back, so all but
  // the first find those rows in L2
  const int nblk = p.Cout / BN;
  const int m0 = (int)(blockIdx.x / nblk) * BM;
  const int n0 = (int)(blockIdx.x % nblk) * BN;

  constexpr bool REQ = FAM == FAM_REQUANT || FAM == FAM_REQUANT_CAPPED;
  const RqPolicy pol = load_channel_block<BN, FAM == FAM_RESIDUAL, FAM == FAM_REQUANT_CAPPED>(p, n0, cs);

  int32_t acc[NACC];

  // RESIDUAL operand tile in shared memory
  const int res_es = (FAM == FAM_RESIDUAL) ? ((p.res_kind == 1 || p.res_bits == 32) ? 4 : 2) : 0;
  const int res_pitch = tile_pitch(BN, res_es);
  uint8_t* sRes = smem + (res_es == 2 ? S::RES16_OFF : S::RES32_OFF);

  auto load_res = [&]() {
    if constexpr (FAM == FAM_RESIDUAL) load_res_tile<BN>(sRes, p, res_es, m0, n0);
  };
  // the uint16 residual operand has its own region: it is fetched while the GEMM runs (the int32 operand overlaps the ring)
  const bool prefetch_res = res_es == 2;

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
      mma_ktile<BN, A4>(acc, smem_u32(sA + stage * S::A_STAGE), smem_u32(sB + stage * S::B_STAGE));
    }
    cp_async_wait<0>();
    __syncthreads();   // pipeline buffers are free
  };

  gemm(ConvGeom{p.x, p.w, p.H, p.W, p.stride, p.pad, p.KH, p.KW, p.cin_chunks, p.x_pix_bytes, p.K}, prefetch_res);

  if (res_es == 4) {   // int32 residual operand: its tile overlaps the ring, so it is loaded now
    load_res();
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
  }
  // the new residual stream is staged in shared memory and written with 16-byte stores, in place over the operand tile when both
  // have the same width
  const bool y_staged = res_es != 0 && p.y_bits == res_es * 8;
  const int y_es = p.y_bits / 8;
  const int y_pitch = tile_pitch(BN, y_es);
  uint8_t* sY = sRes;

  // ------------------------------------------------------------------------------------------------ epilogue
  uint8_t* sOut = smem;
  const bool stage_low = (REQ && p.out_bits <= 8) || (FAM == FAM_RESIDUAL && p.low_bits != 0);
  const int stage_bits = REQ ? p.out_bits : p.low_bits;

  auto put_low = [&](int row, int col, int q0, int q1) { stage_low_pair(sOut, S::OUT_PITCH, row, col, q0, q1); };
  // a pair of the new residual stream, staged or stored directly
  auto put_y = [&](int row, int col, bool ok, int y0, int y1, int& ymax) {
    const uint32_t y16 = p.y_bits == 16 ? stream16_pair(y0, y1, ok, ymax) : 0u;
    if (!y_staged && !ok) return;
    uint8_t* dst = y_staged ? sY + row * y_pitch + col * y_es
                            : reinterpret_cast<uint8_t*>(p.out) + ((size_t)(m0 + row) * p.Cout + n0 + col) * y_es;
    if (p.y_bits == 16) *reinterpret_cast<uint32_t*>(dst) = y16;
    else if (p.y_bits == 32) *reinterpret_cast<int2*>(dst) = make_int2(y0, y1);
  };

  // the REQUANT or RESIDUAL body over one requantisation implementation (RqFp64 or RqExact); REQUANT is compiled separately for
  // 4/8-bit outputs (staged) and 16/32-bit outputs (stored directly), so that no store branch splits the unrolled loop and the
  // terms' FP64 latencies overlap
  auto epilogue = [&](auto rq, auto low_out) {
    if constexpr (REQ) {
      // clamp(RHE((acc + bias) * ratio)), ReLU folded into the lower clamp bound (both implementations are monotone with RHE(0) = 0);
      // capped: the channel's upper clamp from load_channel_block (clamp_hi, or its ReLU6 cap)
      const int lo = p.relu ? min(max(p.lo, 0), p.hi) : p.lo;
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) {
        const int col = fr.col(ni);
        const int4 c0 = *reinterpret_cast<const int4*>(&sChan[col]);   // bias, m, e (capped: upper clamp)
        const int4 c1 = *reinterpret_cast<const int4*>(&sChan[col + 1]);
        const double2 M = *reinterpret_cast<const double2*>(&sM[col]);
        const double2 Cb = *reinterpret_cast<const double2*>(&sCb[col]);
        const int hi0 = FAM == FAM_REQUANT_CAPPED ? c0.w : p.hi, hi1 = FAM == FAM_REQUANT_CAPPED ? c1.w : p.hi;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const int row = fr.row(hf);
          const int q0 = clampi(rq.term(rq.acc_bias(acc[acc_idx(ni, hf)], Cb.x, c0.x), M.x, c0.y, c0.z, false), lo, hi0);
          const int q1 = clampi(rq.term(rq.acc_bias(acc[acc_idx(ni, hf) + 1], Cb.y, c1.x), M.y, c1.y, c1.z, false), lo, hi1);
          if constexpr (decltype(low_out)::value) {
            put_low(row, col, q0, q1);
          } else if (m0 + row < p.M) {
            uint8_t* dst = reinterpret_cast<uint8_t*>(p.out) + ((size_t)(m0 + row) * p.Cout + n0 + col) * (p.out_bits / 8);
            if (p.out_bits == 16) *reinterpret_cast<uint32_t*>(dst) = (uint32_t)(q0 & 0xFFFF) | ((uint32_t)q1 << 16);
            else *reinterpret_cast<int2*>(dst) = make_int2(q0, q1);
          }
        }
      }
    } else {
      // y = [ReLU](sat_add(RHE(r * ratio1), RHE((acc + bias) * ratio))), the new stream and/or the low-bit copy clamp(RHE(y * low ratio))
      const double res_M = dyadic_to_double(p.res_m, p.res_e), low_M = dyadic_to_double(p.low_m, p.low_e);
      const int relu_floor = p.relu ? 0 : (int)0x80000000;
      int ymax = 0;
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) {
        const int col = fr.col(ni);
        const int4 c0 = *reinterpret_cast<const int4*>(&sChan[col]);   // bias, m, e
        const int4 c1 = *reinterpret_cast<const int4*>(&sChan[col + 1]);
        const double2 M = *reinterpret_cast<const double2*>(&sM[col]);
        const double2 Cb = *reinterpret_cast<const double2*>(&sCb[col]);
        double2 M1 = make_double2(res_M, res_M);   // the residual operand's ratio: scalar or per channel
        uint2 m1 = make_uint2(p.res_m, p.res_m);
        int2 e1 = make_int2(p.res_e, p.res_e);
        if (p.res_kind == 1) {
          M1 = *reinterpret_cast<const double2*>(&sM1[col]);
          m1 = make_uint2(sResChan[col].m, sResChan[col + 1].m);
          e1 = make_int2(sResChan[col].e, sResChan[col + 1].e);
        }
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const int row = fr.row(hf);
          const bool ok = m0 + row < p.M;
          const uint8_t* rptr = sRes + row * res_pitch + col * res_es;
          decltype(rq.of_i32(0)) r0, r1;
          if (res_es == 2) {   // uint16 residual stream
            const uint32_t pr = *reinterpret_cast<const uint32_t*>(rptr);
            r0 = rq.of_u16(pr & 0xFFFFu);
            r1 = rq.of_u16(pr >> 16);
          } else {
            const int2 pr = *reinterpret_cast<const int2*>(rptr);
            r0 = rq.of_i32(pr.x);
            r1 = rq.of_i32(pr.y);
          }
          const int y0 = residual_y(rq, rq.term(r0, M1.x, m1.x, e1.x, ok), acc[acc_idx(ni, hf)], Cb.x, c0, M.x, ok, relu_floor);
          const int y1 = residual_y(rq, rq.term(r1, M1.y, m1.y, e1.y, ok), acc[acc_idx(ni, hf) + 1], Cb.y, c1, M.y, ok, relu_floor);
          put_y(row, col, ok, y0, y1, ymax);
          if (p.low_bits != 0) put_low(row, col, residual_low(rq, y0, low_M, p), residual_low(rq, y1, low_M, p));
        }
      }
      residual_flags(p, ymax, rq.ovf);
    }
  };

  if constexpr (FAM == FAM_STORE) {   // RAW_I32: sat_add(acc, bias); DEQUANT_F32: float(acc + bias) * fscale, first cout_store columns
#pragma unroll
    for (int ni = 0; ni < NT; ++ni) {
      const int col = fr.col(ni);
      const int b0 = sChan[col].bias, b1 = sChan[col + 1].bias;
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int m = m0 + fr.row(hf);
        if (m >= p.M) continue;
        const int32_t v0 = sat_add(acc[acc_idx(ni, hf)], b0), v1 = sat_add(acc[acc_idx(ni, hf) + 1], b1);
        if (p.mode == HAWQ_EPI_RAW_I32) {
          *reinterpret_cast<int2*>(reinterpret_cast<int32_t*>(p.out) + (size_t)m * p.Cout + n0 + col) = make_int2(v0, v1);
        } else {
          float* o = reinterpret_cast<float*>(p.out) + (size_t)m * p.cout_store;
          const int c = n0 + col;
          if (c < p.cout_store) o[c] = __fmul_rn((float)v0, p.fscale[c]);
          if (c + 1 < p.cout_store) o[c + 1] = __fmul_rn((float)v1, p.fscale[c + 1]);
        }
      }
    }
  } else {
    auto run = [&](auto low_out) { with_rq<FAM == FAM_RESIDUAL>(pol, p, [&](auto rq) { epilogue(rq, low_out); }); };
    if (REQ && p.out_bits <= 8) run(std::true_type{});
    else run(std::false_type{});
  }

  if (y_staged || stage_low) __syncthreads();
  if (y_staged)   // coalesced copy-out of the new residual stream tile
    copy_out_rows(sY, y_pitch, reinterpret_cast<uint8_t*>(p.out) + (size_t)n0 * y_es, (size_t)p.Cout * y_es, BN * y_es, m0, p.M);
  if (stage_low)
    copy_out_low<BN>(sOut, S::OUT_PITCH, reinterpret_cast<uint8_t*>(REQ ? p.out : p.out_low), stage_bits, m0, n0, p.M, p.Cout);
}

}  // namespace hawq
