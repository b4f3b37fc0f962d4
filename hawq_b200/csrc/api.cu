// C ABI of libhawq_b200.so (see include/hawq_b200.h).  Argument validation + kernel launches; no allocation,
// no synchronisation on the data path (CUDA-graph safe).
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include <cstdlib>

#include "conv_igemm.cuh"
#include "conv_tail.cuh"
#include "elementwise.cuh"
#include "eval_transform.cuh"
#include "mobilenet.cuh"
#include "stem.cuh"

using namespace hawq;

struct hawq_handle {
  int device;
  int sm_count;
  int32_t* status;  // device status word (owned)
};

static thread_local char g_err[512] = "";
static long long g_kernel_count[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // hawq_debug_kernel_count: launches by kernel family (not atomic: debugging aid)

// Sets the thread's hawq_last_error message and returns code; engine_file.cu reports through it too
namespace hawq {
int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
}  // namespace hawq

#define CUDA_TRY(expr)                                                                         \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) return fail(HAWQ_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

static int launch_check(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(HAWQ_ERR_CUDA, "%s launch: %s", what, cudaGetErrorString(e));
  return HAWQ_OK;
}

static int grid_for(long long work_items, int sm_count) {
  long long blocks = (work_items + 255) / 256;
  const long long cap = (long long)sm_count * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

// The maximum carveout lets the driver pick the 228 KB shared-memory configuration, the only one in which two CTAs of every
// conv_igemm and conv_tail instantiation fit (ConvSmem's and TailSmem's static_assert).
template <class K>
static int set_smem_attr(K* kernel, int smem) {
  CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  return HAWQ_OK;
}
template <int BN, bool A4>
static int set_conv_attr() {
  constexpr int smem = ConvSmem<BN, A4>::TOTAL;
  int rc;
  if ((rc = set_smem_attr(conv_igemm_kernel<BN, A4, FAM_REQUANT>, smem)) || (rc = set_smem_attr(conv_igemm_kernel<BN, A4, FAM_RESIDUAL>, smem)) ||
      (rc = set_smem_attr(conv_igemm_kernel<BN, A4, FAM_REQUANT_CAPPED>, smem)) ||
      (rc = set_smem_attr(conv_igemm_kernel<BN, A4, FAM_STORE>, smem)) ||
      (rc = set_smem_attr(conv_tail_kernel<A4, false>, TailSmem<A4, false>::TOTAL)) ||
      (rc = set_smem_attr(conv_tail_kernel<A4, true>, TailSmem<A4, true>::TOTAL)))
    return rc;
  return HAWQ_OK;
}

// 1-D grid of (M / 128 row tiles) x (Cout / BN channel blocks), row tile major (conv_igemm_kernel derives m0, n0)
static dim3 conv_grid(long long M, int Cout, int BN) { return dim3((unsigned)((M + CONV_BM - 1) / CONV_BM * (Cout / BN)), 1, 1); }

template <int BN, bool A4>
static void launch_conv(const ConvParams& p, cudaStream_t s) {
  const int smem = ConvSmem<BN, A4>::TOTAL;
  const dim3 grid = conv_grid(p.M, p.Cout, BN);
  if (p.mode == HAWQ_EPI_REQUANT && p.relu == 2) conv_igemm_kernel<BN, A4, FAM_REQUANT_CAPPED><<<grid, CONV_THREADS, smem, s>>>(p);
  else if (p.mode == HAWQ_EPI_REQUANT) conv_igemm_kernel<BN, A4, FAM_REQUANT><<<grid, CONV_THREADS, smem, s>>>(p);
  else if (p.mode == HAWQ_EPI_RESIDUAL) conv_igemm_kernel<BN, A4, FAM_RESIDUAL><<<grid, CONV_THREADS, smem, s>>>(p);
  else conv_igemm_kernel<BN, A4, FAM_STORE><<<grid, CONV_THREADS, smem, s>>>(p);
}
// persistent tail kernel: bottleneck tails (DUAL = false) and resize units (DUAL = true)
template <bool A4, bool DUAL>
static void launch_conv_tail(const ConvParams& p, int sm_count, cudaStream_t s) {
  conv_tail_kernel<A4, DUAL><<<tail_grid(p.Cout, sm_count), CONV_THREADS, TailSmem<A4, DUAL>::TOTAL, s>>>(p);
}

extern "C" {

int hawq_abi_version(void) { return HAWQ_ABI_VERSION; }
const char* hawq_last_error(void) { return g_err; }

static int create_on(int device, hawq_handle** out) {
  CUDA_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(HAWQ_ERR_UNSUPPORTED, "hawq_create: device sm_%d%d is not Hopper sm_90 (the library is built for sm_90a)", prop.major, prop.minor);
  hawq_handle* h = new hawq_handle();
  h->device = device;
  h->sm_count = prop.multiProcessorCount;
  h->status = nullptr;
  CUDA_TRY(cudaMalloc(&h->status, sizeof(int32_t)));
  CUDA_TRY(cudaMemset(h->status, 0, sizeof(int32_t)));
  int rc;
  CUDA_TRY(cudaFuncSetAttribute(linear_dp4a_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, linear_smem_bytes(LIN_MAX_K)));
  if ((rc = set_conv_attr<128, false>()) || (rc = set_conv_attr<64, false>()) || (rc = set_conv_attr<128, true>()) ||
      (rc = set_conv_attr<64, true>()))
    return rc;
  *out = h;
  return HAWQ_OK;
}

// handles are created per engine, from any thread: the caller's current device is left as it was
int hawq_create(int device, hawq_handle** out) {
  if (!out) return fail(HAWQ_ERR_BAD_ARG, "hawq_create: out is null");
  int prev = 0;
  CUDA_TRY(cudaGetDevice(&prev));
  int rc = create_on(device, out);
  cudaSetDevice(prev);
  return rc;
}

int hawq_destroy(hawq_handle* h) {
  if (!h) return HAWQ_OK;
  cudaFree(h->status);
  delete h;
  return HAWQ_OK;
}

int hawq_sm_count(const hawq_handle* h) { return h ? h->sm_count : 0; }

int hawq_reset_status(hawq_handle* h, void* stream) {
  if (!h) return fail(HAWQ_ERR_BAD_ARG, "null handle");
  CUDA_TRY(cudaMemsetAsync(h->status, 0, sizeof(int32_t), (cudaStream_t)stream));
  return HAWQ_OK;
}

int hawq_get_status(hawq_handle* h, void* stream, int32_t* host_flags) {
  if (!h || !host_flags) return fail(HAWQ_ERR_BAD_ARG, "null argument");
  CUDA_TRY(cudaMemcpyAsync(host_flags, h->status, sizeof(int32_t), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
  return HAWQ_OK;
}

int hawq_copy_status(hawq_handle* h, int32_t* dst, void* stream) {
  if (!h || !dst) return fail(HAWQ_ERR_BAD_ARG, "null argument");
  CUDA_TRY(cudaMemcpyAsync(dst, h->status, sizeof(int32_t), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return HAWQ_OK;
}

// ------------------------------------------------------------------------------------------- argument checks
// Each returns HAWQ_OK or the entry point's error; fn, the entry point's name, prefixes the message.
static int check_me(const char* fn, const char* what, uint32_t m, int e) {
  return e < 1 || e > 62 || m > 0x80000000u ? fail(HAWQ_ERR_BAD_ARG, "%s: %s dyadic pair out of range (m=%u e=%d)", fn, what, m, e) : HAWQ_OK;
}

static int out_size(int in, int k, int stride, int pad) { return (in + 2 * pad - k) / stride + 1; }

// The descriptor of a wgmma convolution; bn: the channel block of the launch's output tiles
static int check_conv_desc(const char* fn, const hawq_conv_desc* d, int bn) {
  if (d->N < 1 || d->H < 1 || d->W < 1 || d->kh < 1 || d->kw < 1 || d->stride < 1 || d->pad < 0) return fail(HAWQ_ERR_BAD_ARG, "%s: bad geometry", fn);
  if (d->a_bits != 8 && d->a_bits != 4) return fail(HAWQ_ERR_UNSUPPORTED, "%s: a_bits must be 4 or 8", fn);
  if (d->Cin % 64 != 0 || d->Cout % 64 != 0) return fail(HAWQ_ERR_UNSUPPORTED, "%s: Cin (%d) and Cout (%d) must be multiples of 64", fn, d->Cin, d->Cout);
  if (d->Cin < 64 || d->Cout < 64) return fail(HAWQ_ERR_BAD_ARG, "%s: Cin (%d) and Cout (%d) must be at least 64", fn, d->Cin, d->Cout);
  const int Ho = out_size(d->H, d->kh, d->stride, d->pad), Wo = out_size(d->W, d->kw, d->stride, d->pad);
  if (Ho < 1 || Wo < 1) return fail(HAWQ_ERR_BAD_ARG, "%s: empty output", fn);
  const long long M = (long long)d->N * Ho * Wo;
  if (M > 0x7fffff00ll || (long long)d->N * d->H * d->W > 0x7fffff00ll) return fail(HAWQ_ERR_UNSUPPORTED, "%s: too many pixels", fn);
  if ((M + CONV_BM - 1) / CONV_BM * (d->Cout / bn) > 0x7fffffffll) return fail(HAWQ_ERR_UNSUPPORTED, "%s: more than 2^31 - 1 output tiles", fn);
  return HAWQ_OK;
}

// The tensors of a direct kernel: at least one image, channel, and row and column (min_side where a stem's window must fit)
static int check_dims(const char* fn, int N, int H, int W, int C, int min_side = 1) {
  return N < 1 || H < min_side || W < min_side || C < 1 ? fail(HAWQ_ERR_BAD_ARG, "%s: bad geometry", fn) : HAWQ_OK;
}

// The launch of a direct kernel: input pixel offsets inside int32, at most 2^31 - 1 CTAs
static int check_limits(const char* fn, long long pixels, long long ctas) {
  if (pixels > 0x7fffff00ll) return fail(HAWQ_ERR_UNSUPPORTED, "%s: too many pixels", fn);
  if (ctas > 0x7fffffffll) return fail(HAWQ_ERR_UNSUPPORTED, "%s: more than 2^31 - 1 CTAs", fn);
  return HAWQ_OK;
}

// A clamp range: not empty, and inside int8 / int16 where `bits` names the stored type
static int check_clamp(const char* fn, int lo, int hi, int bits = 0) {
  if (lo > hi) return fail(HAWQ_ERR_BAD_ARG, "%s: empty clamp range", fn);
  if (bits && (lo < -(1 << (bits - 1)) || hi >= 1 << (bits - 1))) return fail(HAWQ_ERR_BAD_ARG, "%s: clamp must fit int%d", fn, bits);
  return HAWQ_OK;
}

// The low-bit copy clamp(RHE(y * low_m / 2^low_e), low_lo, low_hi): none (low_bits 0), int8 or packed nibbles in out_low
static int check_low(const char* fn, int low_bits, uint32_t low_m, int low_e, const void* out_low) {
  if (low_bits != 0 && low_bits != 4 && low_bits != 8) return fail(HAWQ_ERR_BAD_ARG, "%s: low_bits must be 0/4/8", fn);
  if (!low_bits) return HAWQ_OK;
  if (!out_low) return fail(HAWQ_ERR_BAD_ARG, "%s: low_bits set but out_low is null", fn);
  return check_me(fn, "low-bit copy", low_m, low_e);
}

// The RESIDUAL operand and outputs of an epilogue
static int check_residual(const char* fn, const hawq_epilogue_desc* ep, const void* res, const hawq_chan* res_chan, const void* y,
                          const void* out_low) {
  if (!res) return fail(HAWQ_ERR_BAD_ARG, "%s: RESIDUAL needs res", fn);
  if (ep->res_kind != 0 && ep->res_kind != 1) return fail(HAWQ_ERR_BAD_ARG, "%s: res_kind must be 0/1", fn);
  if (ep->res_kind == 1 && !res_chan) return fail(HAWQ_ERR_BAD_ARG, "%s: res_kind 1 needs res_chan", fn);
  if (ep->res_kind == 0 && ep->res_bits != 16 && ep->res_bits != 32) return fail(HAWQ_ERR_BAD_ARG, "%s: res_bits must be 16/32", fn);
  if (int rc = ep->res_kind == 0 ? check_me(fn, "residual", ep->res_m, ep->res_e) : HAWQ_OK) return rc;
  if (ep->y_bits != 0 && ep->y_bits != 16 && ep->y_bits != 32) return fail(HAWQ_ERR_BAD_ARG, "%s: y_bits must be 0/16/32", fn);
  if (ep->y_bits == 16 && !ep->relu) return fail(HAWQ_ERR_BAD_ARG, "%s: uint16 residual stream requires relu", fn);
  if (ep->y_bits && !y) return fail(HAWQ_ERR_BAD_ARG, "%s: y_bits set but the stream pointer is null", fn);
  if (!ep->y_bits && !ep->low_bits) return fail(HAWQ_ERR_BAD_ARG, "%s: RESIDUAL with no output", fn);
  return check_low(fn, ep->low_bits, ep->low_m, ep->low_e, out_low);
}

// ------------------------------------------------------------------------------------------- kernel parameters
// |acc| <= K * 128 * 128 (int8 activations) or K * 15 * 128 (unsigned 4-bit activations), int8 weights: a bias in
// [bias_lo, bias_hi] keeps acc + bias inside int32, so the FP64 epilogue needs no clamp
static void set_bias_window(ConvParams& p, int a_bits) {
  long long bound = (long long)p.K * (a_bits == 4 ? 15 * 128 : 128 * 128);
  if (bound > 2147483648ll) bound = 2147483648ll;   // empty window: every FP64 CTA clamps acc + bias
  p.bias_lo = (int)(bound - 2147483648ll);
  p.bias_hi = (int)(2147483647ll - bound);
}

// Zeroed parameters of the convolution d with its pointers, geometry and bias window.  K counts the products of one output:
// kh * kw * Cin, or kh * kw in a depthwise convolution (one input channel per output channel).
static ConvParams conv_params(const hawq_handle* h, const hawq_conv_desc& d, const void* x, const int8_t* w, const hawq_chan* chan,
                              void* out, bool depthwise = false) {
  ConvParams p;
  memset(&p, 0, sizeof(p));
  p.x = (const uint8_t*)x; p.w = w; p.chan = chan; p.out = out; p.status = h->status;
  p.N = d.N; p.H = d.H; p.W = d.W; p.Cin = d.Cin; p.Cout = d.Cout; p.KH = d.kh; p.KW = d.kw; p.stride = d.stride; p.pad = d.pad;
  p.Ho = out_size(d.H, d.kh, d.stride, d.pad); p.Wo = out_size(d.W, d.kw, d.stride, d.pad);
  p.M = (int)((long long)d.N * p.Ho * p.Wo); p.K = d.kh * d.kw * (depthwise ? 1 : d.Cin);
  p.cin_chunks = d.Cin / 64; p.x_pix_bytes = d.Cin * d.a_bits / 8;
  set_bias_window(p, d.a_bits);
  return p;
}

// Copies the epilogue into p and derives the scalar part of the kernel's requantisation policy (load_channel_block): whether the scalar
// ratio of a res_kind 0 residual operand or of the low-bit copy exceeds 1 or 2^20, and whether RESIDUAL terms leaving int32 are flagged
// (under a ratio promise).  writes_low: the kernel writes the low-bit copy (RESIDUAL kernels, the stems; not hawq_conv2d's other modes).
static void set_epilogue(ConvParams& p, const hawq_epilogue_desc& ep, bool writes_low) {
  p.mode = ep.mode; p.relu = ep.relu; p.out_bits = ep.out_bits; p.lo = ep.clamp_lo; p.hi = ep.clamp_hi;
  p.res_kind = ep.res_kind; p.res_bits = ep.res_bits; p.res_m = ep.res_m; p.res_e = ep.res_e;
  p.y_bits = ep.y_bits; p.low_bits = ep.low_bits; p.low_m = ep.low_m; p.low_e = ep.low_e; p.low_lo = ep.low_lo; p.low_hi = ep.low_hi;
  p.cout_store = ep.cout_store;
  const bool residual = ep.mode == HAWQ_EPI_RESIDUAL, scalar_res = residual && ep.res_kind == 0;
  const bool low_over_one = writes_low && ep.low_bits != 0 && !dyadic_is_fast(ep.low_m, ep.low_e);
  p.scalar_over_one = (scalar_res && !dyadic_is_fast(ep.res_m, ep.res_e)) || low_over_one;
  p.scalar_unchecked = (scalar_res && !dyadic_is_wide(ep.res_m, ep.res_e)) || low_over_one;
  p.check_ovf = residual && (ep.flags & (HAWQ_EP_RATIOS_LE_ONE | HAWQ_EP_RATIOS_LE_2P20)) != 0;
}

// persistent kernels: 4 CTAs per SM loop over the tiles and stage the weights once (round-2 A/B: 0.212 -> 0.202 ms at batch 128)
static int persistent_ctas(long long tiles, int sm_count) { return (int)(tiles < 4LL * sm_count ? tiles : 4LL * sm_count); }

int hawq_conv2d(hawq_handle* h, const hawq_conv_desc* d, const hawq_epilogue_desc* ep, const void* x, const int8_t* w,
                const hawq_chan* chan, const void* res, const hawq_chan* res_chan, const float* fscale, void* out,
                void* out_low, void* stream) {
  if (!h || !d || !ep || !x || !w || !chan) return fail(HAWQ_ERR_BAD_ARG, "hawq_conv2d: null argument");
  const bool bn128 = (d->Cout % 128 == 0);
  if (int rc = check_conv_desc(__func__, d, bn128 ? 128 : 64)) return rc;
  switch (ep->mode) {
    case HAWQ_EPI_REQUANT:
      if (!out) return fail(HAWQ_ERR_BAD_ARG, "hawq_conv2d: REQUANT needs out");
      if (ep->out_bits != 4 && ep->out_bits != 8 && ep->out_bits != 16 && ep->out_bits != 32)
        return fail(HAWQ_ERR_BAD_ARG, "hawq_conv2d: out_bits must be 4/8/16/32");
      if (int rc = check_clamp(__func__, ep->clamp_lo, ep->clamp_hi)) return rc;
      break;
    case HAWQ_EPI_RESIDUAL:
      if (int rc = check_residual(__func__, ep, res, res_chan, out, out_low)) return rc;
      break;
    case HAWQ_EPI_RAW_I32:
      if (!out) return fail(HAWQ_ERR_BAD_ARG, "hawq_conv2d: RAW_I32 needs out");
      break;
    case HAWQ_EPI_DEQUANT_F32:
      if (!out || !fscale) return fail(HAWQ_ERR_BAD_ARG, "hawq_conv2d: DEQUANT_F32 needs out and fscale");
      if (ep->cout_store < 1 || ep->cout_store > d->Cout) return fail(HAWQ_ERR_BAD_ARG, "hawq_conv2d: bad cout_store");
      break;
    default:
      return fail(HAWQ_ERR_BAD_ARG, "hawq_conv2d: unknown epilogue mode %d", ep->mode);
  }

  ConvParams p = conv_params(h, *d, x, w, chan, out);
  p.res = res; p.res_chan = res_chan; p.fscale = fscale; p.out_low = out_low;
  set_epilogue(p, *ep, ep->mode == HAWQ_EPI_RESIDUAL);
  ++g_kernel_count[0];
  cudaStream_t s = (cudaStream_t)stream;
  // bottleneck tails (1x1 stride 1, uint16 residual operand and stream): the persistent tail kernel
  const bool tail = ep->mode == HAWQ_EPI_RESIDUAL && d->kh == 1 && d->kw == 1 && d->stride == 1 && d->pad == 0 && ep->res_kind == 0 &&
                    ep->res_bits == 16 && ep->y_bits == 16;
  if (tail) {
    if (d->a_bits == 8) launch_conv_tail<false, false>(p, h->sm_count, s);
    else launch_conv_tail<true, false>(p, h->sm_count, s);
  } else if (d->a_bits == 8) {
    if (bn128) launch_conv<128, false>(p, s);
    else launch_conv<64, false>(p, s);
  } else {
    if (bn128) launch_conv<128, true>(p, s);
    else launch_conv<64, true>(p, s);
  }
  return launch_check("conv_igemm");
}

// Resize-unit fusion: y = RHE(m1 * (conv1x1_s(x2, w2) + bias2)) + RHE(m * (conv1x1(x, w) + bias)), ReLU, uint16 stream +
// optional low-bit copy.  Both convolutions run in one kernel (conv_tail.cuh); each thread parks its requantised identity terms in
// shared memory until the main convolution's epilogue (no int32 tensor in HBM).
int hawq_conv2d_dual(hawq_handle* h, const hawq_conv_desc* d, const hawq_epilogue_desc* ep, const void* x, const int8_t* w,
                     const hawq_chan* chan, const hawq_conv_desc* d2, const void* x2, const int8_t* w2, const hawq_chan* chan2,
                     void* out, void* out_low, void* stream) {
  if (!h || !d || !ep || !x || !w || !chan || !d2 || !x2 || !w2 || !chan2 || !out) return fail(HAWQ_ERR_BAD_ARG, "hawq_conv2d_dual: null argument");
  if (d->kh != 1 || d->kw != 1 || d->stride != 1 || d->pad != 0 || d2->kh != 1 || d2->kw != 1 || d2->pad != 0 || d2->stride < 1)
    return fail(HAWQ_ERR_UNSUPPORTED, "hawq_conv2d_dual: both convolutions must be 1x1 without padding (main stride 1)");
  int rc;
  if ((rc = check_conv_desc(__func__, d, 64))) return rc;
  if (d2->a_bits != d->a_bits || d2->Cout != d->Cout) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_conv2d_dual: a_bits and Cout must be equal");
  if (d2->N != d->N || out_size(d2->H, 1, d2->stride, 0) != d->H || out_size(d2->W, 1, d2->stride, 0) != d->W)
    return fail(HAWQ_ERR_BAD_ARG, "hawq_conv2d_dual: the two convolutions have different output grids");
  if ((rc = check_conv_desc(__func__, d2, 64))) return rc;
  if (d->w_layout != 1 || d2->w_layout != 1) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_conv2d_dual: weights must carry the re-tiled copy (w_layout 1)");
  if (ep->mode != HAWQ_EPI_RESIDUAL || !ep->relu || ep->y_bits != 16) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_conv2d_dual: RESIDUAL + relu + uint16 stream only");
  if ((rc = check_low(__func__, ep->low_bits, ep->low_m, ep->low_e, out_low))) return rc;
  if (ep->low_bits && !dyadic_is_fast(ep->low_m, ep->low_e)) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_conv2d_dual: low-bit ratio outside the fast range");
  if (!(ep->flags & (HAWQ_EP_RATIOS_LE_ONE | HAWQ_EP_RATIOS_LE_2P20))) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_conv2d_dual: needs a ratio-range promise (flags)");

  ++g_kernel_count[4];
  ConvParams p = conv_params(h, *d, x, w, chan, out);   // bias window of the main convolution only: the identity operand's bias is added with sat_add
  const ConvParams id = conv_params(h, *d2, x2, w2, chan2, nullptr);
  p.x2 = id.x; p.w2 = id.w; p.H2 = id.H; p.W2 = id.W; p.stride2 = id.stride; p.cin_chunks2 = id.cin_chunks; p.x2_pix_bytes = id.x_pix_bytes;
  p.res_chan = chan2; p.out_low = out_low;
  const hawq_epilogue_desc e = {HAWQ_EPI_RESIDUAL, 1, 0, 0, 0, 1, 32, 0, 0, 16, ep->low_bits, ep->low_m, ep->low_e, ep->low_lo, ep->low_hi, 0, ep->flags};
  set_epilogue(p, e, true);

  cudaStream_t s = (cudaStream_t)stream;
  if (d->a_bits == 8) launch_conv_tail<false, true>(p, h->sm_count, s);
  else launch_conv_tail<true, true>(p, h->sm_count, s);
  return launch_check("conv_dual");
}

int hawq_conv2d_i8(hawq_handle* h, const hawq_conv_desc* d, const hawq_epilogue_desc* ep, const void* x,
                   const int8_t* w, const hawq_chan* chan, const void* res, const hawq_chan* res_chan,
                   const float* fscale, void* out, void* out_low, void* stream) {
  if (d && d->a_bits != 8) return fail(HAWQ_ERR_BAD_ARG, "hawq_conv2d_i8: a_bits must be 8");
  return hawq_conv2d(h, d, ep, x, w, chan, res, res_chan, fscale, out, out_low, stream);
}

int hawq_conv2d_i4(hawq_handle* h, const hawq_conv_desc* d, const hawq_epilogue_desc* ep, const void* x,
                   const int8_t* w, const hawq_chan* chan, const void* res, const hawq_chan* res_chan,
                   const float* fscale, void* out, void* out_low, void* stream) {
  if (d && d->a_bits != 4) return fail(HAWQ_ERR_BAD_ARG, "hawq_conv2d_i4: a_bits must be 4");
  return hawq_conv2d(h, d, ep, x, w, chan, res, res_chan, fscale, out, out_low, stream);
}

int hawq_linear_i8(hawq_handle* h, int32_t N, int32_t K, int32_t Cout, int32_t Cout_pad, const int8_t* x,
                   const int8_t* w, const hawq_chan* chan, const float* fscale, float* out, void* stream) {
  if (Cout < 1 || Cout > Cout_pad) return fail(HAWQ_ERR_BAD_ARG, "hawq_linear_i8: bad Cout/Cout_pad");
  if (!h || !x || !w || !chan || !fscale || !out || N < 1 || K < 1) return fail(HAWQ_ERR_BAD_ARG, "hawq_linear_i8: null argument or empty shape");
  static const bool dp4a_enabled = [] { const char* e = getenv("HAWQ_B200_LINEAR_DP4A"); return !(e && e[0] == '0'); }();
  if (dp4a_enabled && K % LIN_SLAB == 0 && K <= LIN_MAX_K && Cout_pad % LIN_CH == 0 && N <= 65535 * LIN_ROWS) {
    const dim3 grid((unsigned)(Cout_pad / LIN_CH), (unsigned)((N + LIN_ROWS - 1) / LIN_ROWS), 1);
    linear_dp4a_kernel<<<grid, 256, linear_smem_bytes(K), (cudaStream_t)stream>>>(x, w, chan, fscale, out, N, K, Cout);
    return launch_check("linear_dp4a");
  }
  const hawq_conv_desc d = {N, 1, 1, K, Cout_pad, 1, 1, 1, 0, 8, 0};
  hawq_epilogue_desc ep = {};
  ep.mode = HAWQ_EPI_DEQUANT_F32;
  ep.cout_store = Cout;
  return hawq_conv2d(h, &d, &ep, x, w, chan, nullptr, nullptr, fscale, out, nullptr, stream);
}

// ResNet 7x7 / 2 stem (stem.cuh): its channel set-up and requantisation policy are conv_igemm's, over K = 147 int8 products
static ConvParams stem_params(hawq_handle* h, int N, int H, int W, const int8_t* x, const int8_t* w, const hawq_chan* chan,
                              const hawq_epilogue_desc& ep, void* out, void* out_low) {
  ConvParams p = conv_params(h, {N, H, W, 3, 64, 7, 7, 2, 3, 8, 0}, x, w, chan, out);
  p.out_low = out_low;
  set_epilogue(p, ep, true);
  return p;
}

int hawq_stem_conv_i8(hawq_handle* h, int32_t N, int32_t H, int32_t W, const int8_t* x, const int8_t* w,
                      const hawq_chan* chan, int32_t clamp_lo, int32_t clamp_hi, int16_t* out, void* stream) {
  if (!h || !x || !w || !chan || !out) return fail(HAWQ_ERR_BAD_ARG, "hawq_stem_conv_i8: null argument");
  int rc;
  if ((rc = check_dims(__func__, N, H, W, 3, 7)) || (rc = check_clamp(__func__, clamp_lo, clamp_hi, 16))) return rc;
  if (N > 65535) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_stem_conv_i8: N > 65535");
  const ConvParams p = stem_params(h, N, H, W, x, w, chan, {HAWQ_EPI_REQUANT, 1, 0, clamp_lo, clamp_hi}, out, nullptr);
  const dim3 grid((p.Wo + STEM_TW - 1) / STEM_TW, (p.Ho + STEM_TH - 1) / STEM_TH, N);
  stem_conv_kernel<<<persistent_ctas((long long)N * grid.x * grid.y, h->sm_count), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_check("stem_conv");
}

// MobileNetV2 depthwise 3x3 + case-0 requant (mobilenet.cuh); the caps of relu 2 come from chan[c].reserved (load_channel_block)
int hawq_dwconv3x3(hawq_handle* h, int32_t N, int32_t H, int32_t W, int32_t C, int32_t stride, int32_t a_bits, const void* x,
                   const int8_t* w, const hawq_chan* chan, int32_t relu, int32_t out_bits, int32_t clamp_lo, int32_t clamp_hi,
                   void* out, void* stream) {
  if (!h || !x || !w || !chan || !out) return fail(HAWQ_ERR_BAD_ARG, "hawq_dwconv3x3: null argument");
  if (stride != 1 && stride != 2) return fail(HAWQ_ERR_BAD_ARG, "hawq_dwconv3x3: bad geometry");
  int rc;
  if ((rc = check_dims(__func__, N, H, W, C))) return rc;
  if (C % DW_CB != 0) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_dwconv3x3: C (%d) must be a multiple of 16", C);
  if (a_bits != 8 && a_bits != 4) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_dwconv3x3: a_bits must be 4 or 8");
  if (out_bits != 8 && out_bits != 4) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_dwconv3x3: out_bits must be 4 or 8");
  if ((rc = check_clamp(__func__, clamp_lo, clamp_hi))) return rc;
  ConvParams p = conv_params(h, {N, H, W, C, C, 3, 3, stride, 1, a_bits, 0}, x, w, chan, out, true);
  set_epilogue(p, {HAWQ_EPI_REQUANT, relu, out_bits, clamp_lo, clamp_hi}, true);
  const long long strips = (long long)N * ((p.Ho + DW_ROWS - 1) / DW_ROWS) * p.Wo;
  const long long ctas = (strips + DW_THREADS - 1) / DW_THREADS * (C / DW_CB);
  if ((rc = check_limits(__func__, (long long)N * H * W, ctas))) return rc;
  ++g_kernel_count[1];
  if (a_bits == 8) dwconv3x3_kernel<false><<<(unsigned)ctas, DW_THREADS, 0, (cudaStream_t)stream>>>(p);
  else dwconv3x3_kernel<true><<<(unsigned)ctas, DW_THREADS, 0, (cudaStream_t)stream>>>(p);
  return launch_check("dwconv3x3");
}

// MobileNetV2 stem: 3x3 stride 2 pad 1, Cin 3 -> 64 stored channels, requant (+ ReLU6 caps), stream + optional low-bit copy
int hawq_stem3x3_i8(hawq_handle* h, int32_t N, int32_t H, int32_t W, const int8_t* x, const int8_t* w, const hawq_chan* chan, int32_t relu,
                    int32_t clamp_lo, int32_t clamp_hi, int32_t y_bits, void* y, int32_t low_bits, uint32_t low_m, int32_t low_e,
                    int32_t low_lo, int32_t low_hi, void* out_low, void* stream) {
  if (!h || !x || !w || !chan || !y) return fail(HAWQ_ERR_BAD_ARG, "hawq_stem3x3_i8: null argument");
  int rc;
  if ((rc = check_dims(__func__, N, H, W, 3)) || (rc = check_clamp(__func__, clamp_lo, clamp_hi, y_bits == 16 ? 16 : 0))) return rc;
  if (y_bits != 16 && y_bits != 32) return fail(HAWQ_ERR_BAD_ARG, "hawq_stem3x3_i8: y_bits must be 16/32");
  if ((rc = check_low(__func__, low_bits, low_m, low_e, out_low))) return rc;
  ConvParams p = conv_params(h, {N, H, W, 3, 64, 3, 3, 2, 1, 8, 0}, x, w, chan, y);
  p.out_low = out_low;
  set_epilogue(p, {HAWQ_EPI_REQUANT, relu, 0, clamp_lo, clamp_hi, 0, 0, 0, 0, y_bits, low_bits, low_m, low_e, low_lo, low_hi}, true);
  const long long ctas = (long long)N * p.Ho * ((p.Wo + STEM3_PX - 1) / STEM3_PX);
  if ((rc = check_limits(__func__, (long long)N * H * W, ctas))) return rc;
  ++g_kernel_count[2];
  stem3x3_kernel<<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(p);
  return launch_check("stem3x3");
}

int hawq_stem_pool_i8(hawq_handle* h, int32_t N, int32_t H, int32_t W, const int8_t* x, const int8_t* w256, const hawq_chan* chan,
                      int32_t clamp_lo, int32_t clamp_hi, int32_t y_bits, void* y, int32_t low_bits, uint32_t low_m, int32_t low_e,
                      int32_t low_lo, int32_t low_hi, void* out_low, void* stream) {
  if (!h || !x || !w256 || !chan || !y) return fail(HAWQ_ERR_BAD_ARG, "hawq_stem_pool_i8: null argument");
  int rc;
  if ((rc = check_dims(__func__, N, H, W, 3, 7)) || (rc = check_clamp(__func__, clamp_lo, clamp_hi, 16))) return rc;
  if (y_bits != 16 && y_bits != 32) return fail(HAWQ_ERR_BAD_ARG, "hawq_stem_pool_i8: y_bits must be 16/32");
  if ((rc = check_low(__func__, low_bits, low_m, low_e, out_low))) return rc;
  if (W % 16 != 0 || W > 256 || (low_bits && !dyadic_is_fast(low_m, low_e)))
    return fail(HAWQ_ERR_UNSUPPORTED, "hawq_stem_pool_i8: shape / ratio outside the fused kernel (use hawq_stem_conv_i8 + hawq_maxpool_requant)");
  if (N > 65535) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_stem_pool_i8: N > 65535");
  const ConvParams p = stem_params(h, N, H, W, x, w256, chan,
                                   {HAWQ_EPI_REQUANT, 1, 0, clamp_lo, clamp_hi, 0, 0, 0, 0, y_bits, low_bits, low_m, low_e, low_lo, low_hi}, y, out_low);
  const int Po = out_size(p.Ho, 3, 2, 1), Qo = out_size(p.Wo, 3, 2, 1);
  const long long tiles = (long long)N * ((Po + STEMP_PH - 1) / STEMP_PH) * ((Qo + STEMP_PW - 1) / STEMP_PW);
  ++g_kernel_count[6];
  stem_pool_kernel<<<persistent_ctas(tiles, h->sm_count), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_check("stem_pool");
}

int hawq_maxpool_requant(hawq_handle* h, int32_t N, int32_t H, int32_t W, int32_t C, const int16_t* x, int32_t y_bits,
                         void* y, int32_t low_bits, uint32_t low_m, int32_t low_e, int32_t low_lo, int32_t low_hi,
                         void* out_low, void* stream) {
  if (!h || !x) return fail(HAWQ_ERR_BAD_ARG, "hawq_maxpool_requant: null argument");
  if (C % 8 != 0) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_maxpool_requant: C %% 8 != 0");
  if ((y_bits != 0 && y_bits != 16 && y_bits != 32) || (y_bits && !y)) return fail(HAWQ_ERR_BAD_ARG, "hawq_maxpool_requant: bad y");
  int rc;
  if ((rc = check_low(__func__, low_bits, low_m, low_e, out_low)) || (rc = check_dims(__func__, N, H, W, C))) return rc;
  const int Ho = out_size(H, 3, 2, 1), Wo = out_size(W, 3, 2, 1);
  const long long total = (long long)N * Ho * Wo * (C / 8);
  maxpool_requant_kernel<<<grid_for(total, h->sm_count), 256, 0, (cudaStream_t)stream>>>(
      x, N, H, W, C, Ho, Wo, y_bits, y, low_bits, low_m, low_e, low_lo, low_hi, out_low);
  return launch_check("maxpool_requant");
}

int hawq_avgpool_requant(hawq_handle* h, int32_t N, int32_t HW, int32_t C, int32_t x_bits, const void* x, uint32_t m,
                         int32_t e, int32_t lo, int32_t hi, int8_t* out, void* stream) {
  if (!h || !x || !out) return fail(HAWQ_ERR_BAD_ARG, "hawq_avgpool_requant: null argument");
  if (x_bits != 16 && x_bits != 32) return fail(HAWQ_ERR_BAD_ARG, "hawq_avgpool_requant: x_bits must be 16/32");
  int rc;
  if ((rc = check_clamp(__func__, lo, hi, 8)) || (rc = check_me(__func__, "requant", m, e)) || (rc = check_dims(__func__, N, HW, 1, C))) return rc;
  avgpool_requant_kernel<<<grid_for((long long)N * C, h->sm_count), 256, 0, (cudaStream_t)stream>>>(x, N, HW, C, x_bits, m, e, lo, hi, out);
  return launch_check("avgpool_requant");
}

int hawq_quantize_input_f32(hawq_handle* h, int32_t N, int32_t C, int32_t H, int32_t W, const float* x, float scale,
                            int32_t lo, int32_t hi, int8_t* out, void* stream) {
  if (!h || !x || !out) return fail(HAWQ_ERR_BAD_ARG, "hawq_quantize_input_f32: null argument");
  if (!(scale > 0.f)) return fail(HAWQ_ERR_BAD_ARG, "hawq_quantize_input_f32: scale must be > 0");
  if (int rc = check_clamp("hawq_quantize_input_f32", lo, hi, 8)) return rc;
  const float inv = 1.0f / scale;  // fp32 division, as `1. / scale` in linear_quantize (quant_utils.py:97)
  quantize_input_kernel<<<grid_for((long long)N * H * W, h->sm_count), 256, 0, (cudaStream_t)stream>>>(x, N, C, H, W, inv, lo, hi, out);
  return launch_check("quantize_input");
}

int hawq_quantize_input_u8(hawq_handle* h, int32_t N, int32_t H, int32_t W, const uint8_t* x, const float* mean3,
                           const float* std3, float scale, int32_t lo, int32_t hi, int8_t* out, void* stream) {
  if (!h || !x || !out || !mean3 || !std3) return fail(HAWQ_ERR_BAD_ARG, "hawq_quantize_input_u8: null argument");
  int rc;
  if ((rc = check_dims(__func__, N, H, W, 3))) return rc;
  if (!(scale > 0.f)) return fail(HAWQ_ERR_BAD_ARG, "hawq_quantize_input_u8: scale must be > 0");
  if ((rc = check_clamp(__func__, lo, hi, 8))) return rc;
  for (int c = 0; c < 3; ++c)
    if (!(std3[c] > 0.f)) return fail(HAWQ_ERR_BAD_ARG, "hawq_quantize_input_u8: std must be > 0");
  const float inv = 1.0f / scale;  // fp32 division, as `1. / scale` in linear_quantize (quant_utils.py:97)
  const long long n_bytes = (long long)N * H * W * 3;
  quantize_input_u8_kernel<<<grid_for(n_bytes / 4 + 1, h->sm_count), 256, 0, (cudaStream_t)stream>>>(
      x, n_bytes, 3, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2], inv, lo, hi, out);
  return launch_check("quantize_input_u8");
}

int hawq_resize_crop_quantize_u8(hawq_handle* h, int32_t B, const uint8_t* pixels, int64_t pixel_bytes, const hawq_image_desc* table,
                                 int32_t S, int32_t Ch, int32_t Cw, const float* mean3, const float* std3, float scale, int32_t lo,
                                 int32_t hi, int8_t* out, void* stream) {
  if (!h || !pixels || !table || !out || !mean3 || !std3) return fail(HAWQ_ERR_BAD_ARG, "hawq_resize_crop_quantize_u8: null argument");
  if (B < 1 || B > 65535) return fail(HAWQ_ERR_BAD_ARG, "hawq_resize_crop_quantize_u8: B = %d outside 1..65535", B);
  if (Ch < 1 || Cw < 1 || pixel_bytes < 0) return fail(HAWQ_ERR_BAD_ARG, "hawq_resize_crop_quantize_u8: empty crop or negative arena");
  if (S < ET_MIN_RESIZE || S > ET_MAX_SIDE || S < Ch || S < Cw)
    return fail(HAWQ_ERR_UNSUPPORTED, "hawq_resize_crop_quantize_u8: resize %d must lie in %d..%d and cover the crop %dx%d", S,
                ET_MIN_RESIZE, ET_MAX_SIDE, Ch, Cw);
  if (!(scale > 0.f)) return fail(HAWQ_ERR_BAD_ARG, "hawq_resize_crop_quantize_u8: scale must be > 0");
  if (int rc = check_clamp("hawq_resize_crop_quantize_u8", lo, hi, 8)) return rc;
  for (int c = 0; c < 3; ++c)
    if (!(std3[c] > 0.f)) return fail(HAWQ_ERR_BAD_ARG, "hawq_resize_crop_quantize_u8: std must be > 0");
  const float inv = 1.0f / scale;  // as hawq_quantize_input_u8
  const dim3 grid((Cw + ET_TW - 1) / ET_TW, (Ch + ET_TR - 1) / ET_TR, B);
  resize_crop_quantize_u8_kernel<<<grid, ET_THREADS, 0, (cudaStream_t)stream>>>(pixels, pixel_bytes, table, S, Ch, Cw, mean3[0], mean3[1],
                                                                                  mean3[2], std3[0], std3[1], std3[2], inv, lo, hi, out);
  return launch_check("resize_crop_quantize_u8");
}

int hawq_requant(hawq_handle* h, int64_t rows, int32_t C, int32_t x_bits, const void* x, const hawq_chan* chan,
                 int32_t chan_stride, int32_t relu, int32_t out_bits, int32_t lo, int32_t hi, void* out, void* stream) {
  if (!h || !x || !chan || !out) return fail(HAWQ_ERR_BAD_ARG, "hawq_requant: null argument");
  if (C % 8 != 0) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_requant: C %% 8 != 0");
  if (x_bits != 16 && x_bits != 32) return fail(HAWQ_ERR_BAD_ARG, "hawq_requant: x_bits must be 16/32");
  if (out_bits != 4 && out_bits != 8 && out_bits != 16 && out_bits != 32) return fail(HAWQ_ERR_BAD_ARG, "hawq_requant: out_bits must be 4/8/16/32");
  if (chan_stride != 0 && chan_stride != 1) return fail(HAWQ_ERR_BAD_ARG, "hawq_requant: chan_stride must be 0/1");
  if (int rc = check_clamp("hawq_requant", lo, hi)) return rc;
  requant_kernel<<<grid_for(rows * (C / 8), h->sm_count), 256, 0, (cudaStream_t)stream>>>(x, rows, C, x_bits, chan, chan_stride, relu, out_bits, lo, hi, out);
  return launch_check("requant");
}

int hawq_add_requant(hawq_handle* h, int64_t rows, int32_t C, const int32_t* acc, const hawq_chan* chan,
                     const hawq_epilogue_desc* ep, const void* res, const hawq_chan* res_chan, void* y, void* out_low,
                     void* stream) {
  if (!h || !acc || !chan || !ep || !res) return fail(HAWQ_ERR_BAD_ARG, "hawq_add_requant: null argument");
  if (C % 8 != 0) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_add_requant: C %% 8 != 0");
  if (int rc = check_residual("hawq_add_requant", ep, res, res_chan, y, out_low)) return rc;
  AddRequantParams p;
  p.acc = acc; p.chan = chan; p.res = res; p.res_chan = res_chan; p.y = y; p.out_low = out_low; p.status = h->status;
  p.rows = rows; p.C = C; p.relu = ep->relu; p.res_kind = ep->res_kind; p.res_bits = ep->res_bits; p.res_m = ep->res_m;
  p.res_e = ep->res_e; p.y_bits = ep->y_bits; p.low_bits = ep->low_bits; p.low_m = ep->low_m; p.low_e = ep->low_e;
  p.low_lo = ep->low_lo; p.low_hi = ep->low_hi;
  add_requant_kernel<<<grid_for(rows * (C / 8), h->sm_count), 256, 0, (cudaStream_t)stream>>>(p);
  return launch_check("add_requant");
}

int hawq_dequant_f32(hawq_handle* h, int32_t N, int32_t H, int32_t W, int32_t C, int32_t x_bits, int32_t x_signed,
                     const void* x, float scale, float* out_nchw, void* stream) {
  if (!h || !x || !out_nchw) return fail(HAWQ_ERR_BAD_ARG, "hawq_dequant_f32: null argument");
  if (x_bits != 4 && x_bits != 8 && x_bits != 16 && x_bits != 32) return fail(HAWQ_ERR_BAD_ARG, "hawq_dequant_f32: bad x_bits");
  if (x_bits == 4 && C % 8 != 0) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_dequant_f32: packed input needs C %% 8 == 0");
  dequant_f32_kernel<<<grid_for((long long)N * H * W * C, h->sm_count), 256, 0, (cudaStream_t)stream>>>(x, N, H, W, C, x_bits, x_signed, scale, out_nchw);
  return launch_check("dequant_f32");
}

int hawq_pack_i4(hawq_handle* h, int64_t n_values, const uint8_t* in, uint8_t* out, void* stream) {
  if (!h || !in || !out || n_values % 8 != 0) return fail(HAWQ_ERR_BAD_ARG, "hawq_pack_i4: bad argument");
  pack_i4_kernel<<<grid_for(n_values / 8, h->sm_count), 256, 0, (cudaStream_t)stream>>>(in, n_values / 8, out);
  return launch_check("pack_i4");
}

int hawq_unpack_i4(hawq_handle* h, int64_t n_values, const uint8_t* in, uint8_t* out, void* stream) {
  if (!h || !in || !out || n_values % 8 != 0) return fail(HAWQ_ERR_BAD_ARG, "hawq_unpack_i4: bad argument");
  unpack_i4_kernel<<<grid_for(n_values / 8, h->sm_count), 256, 0, (cudaStream_t)stream>>>(in, n_values / 8, out);
  return launch_check("unpack_i4");
}

// ------------------------------------------------------------------------------------------- host helpers
int hawq_dyadic(double ratio, uint32_t* m, int32_t* e) {
  if (!m || !e || !(ratio > 0.0) || !std::isfinite(ratio)) return fail(HAWQ_ERR_BAD_ARG, "hawq_dyadic: ratio must be positive and finite");
  int ex;
  const double mant = std::frexp(ratio, &ex);          // mant in [0.5, 1)
  const double scaled = mant * 2147483648.0;            // exact
  const double r = std::floor(scaled + 0.5);            // ROUND_HALF_UP for positive values, exact (see oracle/int_ref.py)
  const int ee = 31 - ex;
  if (ee < 1) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_dyadic: ratio %g too large (e = %d < 1)", ratio, ee);
  if (ee > 62) { *m = 0; *e = 1; return HAWQ_OK; }      // |v*m| < 2^62 <= 2^(e-1): always rounds to 0
  *m = (uint32_t)r;
  *e = ee;
  return HAWQ_OK;
}

int64_t hawq_rhe_requant_host(int32_t v, uint32_t m, int32_t e) { return (int64_t)rhe_requant(v, m, e); }

int hawq_permute_weights_for_i4(int8_t* host_w, int64_t rows_times_taps, int32_t Cin) {
  if (!host_w || Cin % 32 != 0) return fail(HAWQ_ERR_BAD_ARG, "hawq_permute_weights_for_i4: Cin %% 32 != 0");
  int8_t tmp[32];
  for (int64_t r = 0; r < rows_times_taps; ++r) {
    for (int blk = 0; blk < Cin / 32; ++blk) {
      int8_t* p = host_w + r * Cin + blk * 32;
      for (int t = 0; t < 4; ++t)
        for (int j = 0; j < 4; ++j) {
          tmp[4 * t + j] = p[8 * t + j];           // MMA k position 4t+j     <- channel 8t+j
          tmp[16 + 4 * t + j] = p[8 * t + 4 + j];  // MMA k position 16+4t+j  <- channel 8t+4+j
        }
      memcpy(p, tmp, 32);
    }
  }
  return HAWQ_OK;
}

int64_t hawq_workspace_bytes(const hawq_conv_desc*, const hawq_epilogue_desc*) { return 0; }

int hawq_retile_weights(hawq_handle* h, const int8_t* w_ohwi, int32_t Cout, int64_t K, int8_t* out, void* stream) {
  if (!h || !w_ohwi || !out) return fail(HAWQ_ERR_BAD_ARG, "hawq_retile_weights: null argument");
  if (Cout % 64 != 0 || K % 64 != 0) return fail(HAWQ_ERR_UNSUPPORTED, "hawq_retile_weights: Cout and K must be multiples of 64");
  const int bn = (Cout % 128 == 0) ? 128 : 64;
  const long long chunks = (long long)Cout * K / 16;
  retile_weights_kernel<<<grid_for(chunks, h->sm_count), 256, 0, (cudaStream_t)stream>>>(w_ohwi, Cout, (int)K, bn, out);
  return launch_check("retile_weights");
}


int64_t hawq_debug_kernel_count(int32_t family) { return (family >= 0 && family < 8) ? g_kernel_count[family] : -1; }

}  // extern "C"
