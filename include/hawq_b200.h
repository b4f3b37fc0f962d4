/* hawq_b200.h — C ABI of libhawq_b200.so: the integer forward path of HAWQ-quantized ResNets on H100 (sm_90a).
 *
 * The reference (Zhen-Dong/HAWQ) has no FFI / operator-registration layer: its boundary for this path is the Python
 * nn.Module API of utils/quantization_utils/quant_modules.py.  Each entry point below therefore cites the reference
 * *module/function* whose frozen (eval) forward it replaces; hawq_b200/ (Python) mirrors the module API on top of
 * this ABI, INTEGRATION.md shows the ctypes binding.
 *
 * Conventions
 *   - plain pointers + sizes, no torch types; all pointers are DEVICE pointers unless named host_*;
 *   - every call is asynchronous on the caller-supplied stream (cudaStream_t passed as void*), never allocates,
 *     never synchronises -> safe under CUDA-graph capture;
 *   - return value: 0 = HAWQ_OK, negative = hawq_status; hawq_last_error() gives a thread-local message;
 *   - every device pointer must be 16-byte aligned (the kernels move activations, weights and outputs in 16-byte vectors);
 *   - a call writes exactly the elements of its outputs and nothing else: a packed 4-bit output is numel / 2 bytes, DEQUANT_F32
 *     writes rows of cout_store floats, hawq_linear_i8 writes N x Cout floats.  It never writes its inputs, and it neither reads
 *     nor writes a pointer its arguments leave unused (res / res_chan / fscale / out_low of an epilogue that does not take them,
 *     out with y_bits 0, out_low with low_bits 0), so such a pointer may be null or point anywhere;
 *   - activations are NHWC.  8-bit: one int8 per element.  4-bit: unsigned nibbles packed two per byte in the
 *     "hawq nibble order": inside every group of 8 consecutive channels, byte j (0..3) holds channel j in its low
 *     nibble and channel j+4 in its high nibble (so a 32-bit word expands to two int8x4 words with one AND and one
 *     SHIFT+AND).  hawq_pack_i4 / hawq_unpack_i4 convert from/to one-value-per-byte;
 *   - weights are int8, OHWI ([Cout][kh][kw][Cin], K-major) for 8- and 4-bit layers alike (Hopper has no int4
 *     MMA: 4-bit weights are widened once at plan time; they are <1% of the traffic).  For layers whose INPUT is
 *     packed 4-bit the K order inside each 32-channel block must be permuted with hawq_permute_weights_for_i4
 *     (host helper) to match the on-chip nibble expansion;
 *   - the residual stream ("x16": the output of quant_act_int32, reference utils/models/q_resnet.py:120,254-258)
 *     is stored post-ReLU either as int32 (always exact) or as uint16 with saturation + sticky overflow flag
 *     (HAWQ_FLAG_RESIDUAL_OVERFLOW in the handle's status word; the host re-runs with int32 when it is set);
 *   - dyadic requantisation everywhere is q = RHE(v * m / 2^e), round-half-to-EVEN, i.e. the reference's
 *     torch.round(f64(v)*f64(m)/2^e) (utils/quantization_utils/quant_utils.py:406-408), with (m, e) from
 *     batch_frexp (quant_utils.py:188-213): 2^30 <= m <= 2^31, 1 <= e <= 62.
 */
#ifndef HAWQ_B200_H
#define HAWQ_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HAWQ_ABI_VERSION 1

typedef struct hawq_handle hawq_handle;

enum hawq_status {
  HAWQ_OK = 0,
  HAWQ_ERR_BAD_ARG = -1,      /* null pointer, non-positive size, inconsistent descriptor */
  HAWQ_ERR_UNSUPPORTED = -2,  /* shape / bit-width combination this build has no kernel for */
  HAWQ_ERR_CUDA = -3,         /* CUDA runtime error (message in hawq_last_error) */
  HAWQ_ERR_RESULT_INVALID = -4 /* hawq_engine_run: HAWQ_FLAG_BAD_RATIO was raised, the logits are invalid */
};

/* bits of the device status word */
#define HAWQ_FLAG_RESIDUAL_OVERFLOW 1   /* a post-ReLU residual value exceeded 65535 while stored as uint16 */
#define HAWQ_FLAG_BAD_RATIO 2           /* a HAWQ_EP_RATIOS_* promise was broken: results invalid */
#define HAWQ_FLAG_REQUANT_OVERFLOW 4     /* a requantised value left int32 on the fast path (ratio > 1): re-run without HAWQ_EP_* flags */

/* Per-output-channel epilogue parameters (16 B, one vector load per channel).
 * bias = bias_integer (quant_modules.py:481-484), (m, e) = batch_frexp of the requant ratio of that channel.
 * reserved: with relu 2 (ReLU6) in a REQUANT epilogue, hawq_dwconv3x3 or hawq_stem3x3_i8 it is the channel's output cap: the
 * upper clamp of channel c is min(clamp_hi, reserved), so q = max(lo', min(RHE(...), min(clamp_hi, reserved))) with the ReLU-folded
 * lo' = min(max(clamp_lo, 0), clamp_hi).  ReLU6 (q_mobilenetv2.py) caps the accumulator at C_c = round_f32(6 / a_sf / w_sf_c), and the
 * requantisation is monotone, so reserved = RHE(C_c * m_c / 2^e_c) (hawq_rhe_requant_host; clamp_hi when C_c >= 2^31).  With relu 0
 * or 1 it means nothing. */
typedef struct {
  int32_t bias;
  uint32_t m;
  int32_t e;
  int32_t reserved;
} hawq_chan;

/* Convolution geometry.  Replaces the F.conv2d call of QuantBnConv2d.forward / QuantConv2d.forward
 * (quant_modules.py:493, :731-736).  Requirements: Cin % 64 == 0, Cout % 64 == 0 (pad on the host otherwise). */
typedef struct {
  int32_t N, H, W, Cin, Cout;
  int32_t kh, kw, stride, pad;
  int32_t a_bits;    /* 8: int8 NHWC input; 4: packed unsigned nibbles (hawq nibble order) */
  int32_t w_layout;  /* 0: w = OHWI only; 1: w = OHWI followed by the hawq_retile_weights copy (2 * Cout * K bytes) */
} hawq_conv_desc;

enum hawq_epilogue_mode {
  HAWQ_EPI_REQUANT = 0,   /* case 0, fixedpoint_fn (quant_utils.py:390-413): clamp(RHE((acc+bias)[relu] * m_c / 2^e_c)) */
  HAWQ_EPI_RESIDUAL = 1,  /* case 1 (quant_utils.py:416-456): RHE(res*m1/2^e1) + RHE((acc+bias)*m_c/2^e_c), no clamp, [relu] */
  HAWQ_EPI_RAW_I32 = 2,   /* acc + bias as int32 (identity-branch conv feeding case 1) */
  HAWQ_EPI_DEQUANT_F32 = 3 /* QuantLinear tail (quant_modules.py:129-130): float(acc+bias) * fscale[c] */
};

typedef struct {
  int32_t mode;           /* hawq_epilogue_mode */
  int32_t relu;           /* REQUANT: 1 = max(acc+bias,0) before requant, 2 = that and the per-channel ReLU6 cap of hawq_chan.reserved;
                             RESIDUAL: max(sum,0) after the add */
  /* REQUANT output */
  int32_t out_bits;       /* 4 (packed u4), 8 (int8), 16 (int16), 32 (int32) */
  int32_t clamp_lo, clamp_hi;
  /* RESIDUAL input operand */
  int32_t res_kind;       /* 0: residual-stream tensor, scalar (res_m, res_e); 1: int32 accumulator tensor, per-channel res_chan */
  int32_t res_bits;       /* res_kind 0: 16 (uint16) or 32 (int32) */
  uint32_t res_m;
  int32_t res_e;
  /* RESIDUAL outputs */
  int32_t y_bits;         /* 0: do not store the new residual stream; 16: uint16 (needs relu=1); 32: int32 */
  int32_t low_bits;       /* 0: none; 4 / 8: also store clamp(RHE(y * low_m / 2^low_e)) = the next quant_act's output */
  uint32_t low_m;
  int32_t low_e;
  int32_t low_lo, low_hi;
  /* DEQUANT_F32 */
  int32_t cout_store;     /* number of real output columns (<= Cout), row pitch of the fp32 output */
  int32_t flags;          /* HAWQ_EP_*: promises of the caller that unlock faster kernels */
} hawq_epilogue_desc;

/* Caller promise: every dyadic pair of this launch (chan[], res_chan[], res_m/e, low_m/e) has ratio m * 2^-e <= 1, i.e.
 * e >= 31 or m == 0 (true for every HAWQ ResNet layer).  The convolution evaluates RHE(v * m / 2^e) with one exact FP64 FMA
 * when every ratio of the CTA's channels is <= 1 (checked in the kernel) and with the exact 64-bit integer form otherwise. */
#define HAWQ_EP_RATIOS_LE_ONE 1
/* Weaker promise: every ratio <= 2^20 (e >= 11 or m == 0).  Under either promise a RESIDUAL term whose requantised value
 * leaves int32 raises HAWQ_FLAG_REQUANT_OVERFLOW (without a promise the sum saturates silently, as the reference's int32 cast). */
#define HAWQ_EP_RATIOS_LE_2P20 2

/* ---- lifetime ---------------------------------------------------------------------------------------------- */
int hawq_abi_version(void);
const char* hawq_last_error(void);
int hawq_create(int device, hawq_handle** out);
int hawq_destroy(hawq_handle* h);
int hawq_sm_count(const hawq_handle* h);
/* status word (sticky flags set by kernels): reset is async on the stream, get synchronises the stream */
int hawq_reset_status(hawq_handle* h, void* stream);
int hawq_get_status(hawq_handle* h, void* stream, int32_t* host_flags);
/* async copy of the status word into a caller-owned device int32 (e.g. inside a CUDA graph) */
int hawq_copy_status(hawq_handle* h, int32_t* dst, void* stream);

/* ---- fused convolution (QuantBnConv2d / QuantConv2d + the QuantAct that consumes it) ------------------------- */
/* x: activations (int8 or packed u4, NHWC); w: int8 OHWI; chan[Cout];
 * res / res_chan: RESIDUAL operand (see res_kind); fscale[Cout]: DEQUANT_F32;
 * out: REQUANT result | RAW int32 | fp32 logits | new residual stream (RESIDUAL, y_bits != 0);
 * out_low: RESIDUAL low-bit copy (low_bits != 0). */
int hawq_conv2d(hawq_handle* h, const hawq_conv_desc* d, const hawq_epilogue_desc* ep,
                const void* x, const int8_t* w, const hawq_chan* chan,
                const void* res, const hawq_chan* res_chan, const float* fscale,
                void* out, void* out_low, void* stream);
/* the two names SURVEY.md §8(b) proposes; thin checks over hawq_conv2d (a_bits must be 8 resp. 4) */
int hawq_conv2d_i8(hawq_handle* h, const hawq_conv_desc* d, const hawq_epilogue_desc* ep,
                   const void* x, const int8_t* w, const hawq_chan* chan,
                   const void* res, const hawq_chan* res_chan, const float* fscale,
                   void* out, void* out_low, void* stream);
int hawq_conv2d_i4(hawq_handle* h, const hawq_conv_desc* d, const hawq_epilogue_desc* ep,
                   const void* x, const int8_t* w, const hawq_chan* chan,
                   const void* res, const hawq_chan* res_chan, const float* fscale,
                   void* out, void* out_low, void* stream);

/* Resize residual units (Q_ResUnitBn with resize_identity, q_resnet.py:304-330): the identity-branch 1x1 convolution
 * (d2/x2/w2; stride d2->stride, pad 0) and the unit's last 1x1 convolution (d/x/w; stride 1) are computed one after the other
 * in one kernel (the identity result stays in shared memory) and combined by the case-1 fixed-point sum (quant_utils.py:430-456):
 *   y = ReLU( RHE((acc2 + chan2.bias) * chan2.m / 2^chan2.e) + RHE((acc + chan.bias) * chan.m / 2^chan.e) )
 * ep: mode RESIDUAL, relu 1, y_bits 16 (uint16 stream in out), optional low-bit copy in out_low, flags = ratio promise.
 * Both descriptors need w_layout 1 and equal a_bits / Cout / output grids.  Returns HAWQ_ERR_UNSUPPORTED for any other
 * combination (callers then use hawq_conv2d RAW_I32 followed by hawq_conv2d RESIDUAL res_kind 1: same results). */
int hawq_conv2d_dual(hawq_handle* h, const hawq_conv_desc* d, const hawq_epilogue_desc* ep,
                     const void* x, const int8_t* w, const hawq_chan* chan,
                     const hawq_conv_desc* d2, const void* x2, const int8_t* w2, const hawq_chan* chan2,
                     void* out, void* out_low, void* stream);

/* QuantLinear.forward (quant_modules.py:79-130): x int8 [N,K], w int8 [Cout_pad,K] (rows >= Cout zero),
 * chan[Cout_pad] (bias only), fscale[Cout_pad] = fc_scaling_factor[c] * act_scale (fp32 product) -> fp32 [N,Cout]. */
int hawq_linear_i8(hawq_handle* h, int32_t N, int32_t K, int32_t Cout, int32_t Cout_pad,
                   const int8_t* x, const int8_t* w, const hawq_chan* chan, const float* fscale,
                   float* out, void* stream);

/* ---- stem: 7x7 s2 p3 conv, Cin = 3 (Q_ResNet*.quant_init*_convbn, q_resnet.py:117) -------------------------- */
/* x int8 [N,H,W,3]; w int8 [64][7][8][4] (kw 7 and channel 3 zero); chan[64] carries bias and the 16-bit requant of
 * quant_act_int32 (q_resnet.py:120).  Output int16 [N,Ho,Wo,64] = max(0, clamp(RHE((acc+bias)*m/2^e), lo, hi)):
 * requant and ReLU commute with the max-pool that follows (both monotone). */
int hawq_stem_conv_i8(hawq_handle* h, int32_t N, int32_t H, int32_t W, const int8_t* x, const int8_t* w,
                      const hawq_chan* chan, int32_t clamp_lo, int32_t clamp_hi, int16_t* out, void* stream);

/* Fused stem: quant_init_convbn (7x7 stride 2 pad 3, Cin = 3 -> 64) + nn.MaxPool2d(3, 2, 1) + quant_act_int32 (16-bit dyadic
 * requant, clamp) + ReLU, and optionally the first unit's low-bit quant_act (q_resnet.py:117-122, :234) in one kernel; the int16
 * convolution output never reaches HBM.  w256 = int8 [64][8][8][4] (kernel rows padded 7 -> 8, taps 7 -> 8, channels 3 -> 4, zeros
 * in the padding).  y = pooled residual stream [N][Hp][Wp][64] as uint16 (y_bits 16) or int32 (32).  Preconditions: the ratio
 * of the low-bit copy <= 1, W % 16 == 0 (row pitch a multiple of 16 bytes), W <= 256; otherwise HAWQ_ERR_UNSUPPORTED (use
 * hawq_stem_conv_i8 + hawq_maxpool_requant: same integers). */
int hawq_stem_pool_i8(hawq_handle* h, int32_t N, int32_t H, int32_t W, const int8_t* x, const int8_t* w256, const hawq_chan* chan,
                      int32_t clamp_lo, int32_t clamp_hi, int32_t y_bits, void* y, int32_t low_bits, uint32_t low_m, int32_t low_e,
                      int32_t low_lo, int32_t low_hi, void* out_low, void* stream);
/* nn.MaxPool2d(3,2,1) (q_resnet.py:119) on the int16 stem output + the first unit's quant_act (case 0, scalar m,e).
 * Precondition: 0 <= x <= 32767 (the post-ReLU stem output); the kernel pads with 0 and reads the maxima as unsigned, so
 * negative inputs give unspecified results.
 * y: residual stream (y_bits 16 -> uint16, 32 -> int32); out_low: int8 / packed u4 (low_bits 8 / 4, 0 = none).
 * Requires N, H, W, C >= 1, y_bits 0 / 16 / 32, low_bits 0 / 4 / 8 (1 <= low_e <= 62, low_m <= 2^31) and C % 8 == 0 (else
 * HAWQ_ERR_UNSUPPORTED); a call outside these returns HAWQ_ERR_BAD_ARG and launches nothing. */
int hawq_maxpool_requant(hawq_handle* h, int32_t N, int32_t H, int32_t W, int32_t C, const int16_t* x,
                         int32_t y_bits, void* y, int32_t low_bits, uint32_t low_m, int32_t low_e,
                         int32_t low_lo, int32_t low_hi, void* out_low, void* stream);

/* ---- MobileNetV2 (reference utils/models/q_mobilenetv2.py) --------------------------------------------------- */
/* Depthwise 3x3 convolution, pad 1, stride 1 or 2 (Q_LinearBottleneck.conv2, groups = C) + the QuantAct that consumes it (case 0,
 * per-channel chan[C], relu 0 / 1 / 2 as in hawq_epilogue_desc).  x: NHWC [N,H,W,C], int8 (a_bits 8; 4-bit values 0..15 in byte
 * containers too) or packed nibbles (a_bits 4); w: int8 [3][3][C] (channel-minor); C % 16 == 0.
 * out [N,Ho,Wo,C]: int8 (out_bits 8) or packed nibbles (out_bits 4) of max(lo', min(RHE((acc + bias) * m_c / 2^e_c), hi_c)). */
int hawq_dwconv3x3(hawq_handle* h, int32_t N, int32_t H, int32_t W, int32_t C, int32_t stride, int32_t a_bits, const void* x,
                   const int8_t* w, const hawq_chan* chan, int32_t relu, int32_t out_bits, int32_t clamp_lo, int32_t clamp_hi,
                   void* out, void* stream);
/* MobileNetV2 stem (init_block: 3x3 stride 2 pad 1, Cin 3) + quant_act_int32 (case 0, relu 0 / 1 / 2 as in hawq_epilogue_desc).
 * x int8 [N,H,W,3]; w int8 [64][3][3][4] (channel 3 zero; a model with fewer output channels pads with zero rows and m = 0);
 * chan[64].  y [N,Ho,Wo,64]: int16 (y_bits 16, clamp inside int16) or int32 (32).  Optionally the next QuantAct's copy
 * clamp(RHE(y * low_m / 2^low_e), low_lo, low_hi) as int8 / packed nibbles (low_bits 8 / 4, 0 = none). */
int hawq_stem3x3_i8(hawq_handle* h, int32_t N, int32_t H, int32_t W, const int8_t* x, const int8_t* w, const hawq_chan* chan, int32_t relu,
                    int32_t clamp_lo, int32_t clamp_hi, int32_t y_bits, void* y, int32_t low_bits, uint32_t low_m, int32_t low_e,
                    int32_t low_lo, int32_t low_hi, void* out_low, void* stream);

/* QuantAveragePool2d (quant_modules.py:585-602) + quant_act_output (q_resnet.py:131): x residual stream
 * [N,HW,C] (x_bits 16/32) -> int8 [N,C] = clamp(RHE(trunc_avg(x) * m / 2^e)).
 * Requires N, HW, C >= 1, -128 <= lo <= hi <= 127, 1 <= e <= 62 and m <= 2^31; otherwise HAWQ_ERR_BAD_ARG (nothing launched). */
int hawq_avgpool_requant(hawq_handle* h, int32_t N, int32_t HW, int32_t C, int32_t x_bits, const void* x,
                         uint32_t m, int32_t e, int32_t lo, int32_t hi, int8_t* out, void* stream);

/* ---- stand-alone (unfused) pieces of the module API --------------------------------------------------------- */
/* QuantAct input branch (quant_modules.py:271-274): q = clamp(round((1/scale) * x)), fp32 RNE.
 * x fp32 NCHW [N,C,H,W] -> int8 NHWC [N,H,W,C].  +-inf clamp to lo / hi.  NaN is outside the reference's semantics (its
 * integer cast of NaN is undefined): the result for a NaN element is unspecified.  Requires scale > 0 and -128 <= lo <= hi <= 127
 * (else HAWQ_ERR_BAD_ARG, nothing launched). */
int hawq_quantize_input_f32(hawq_handle* h, int32_t N, int32_t C, int32_t H, int32_t W, const float* x,
                            float scale, int32_t lo, int32_t hi, int8_t* out, void* stream);
/* uint8 image entry (tvm_benchmark/test_resnet_accuracy_imagenet.py:62-75 quantize_image after transforms.ToTensor + Normalize
 * :82-93): x uint8 NHWC [N,H,W,3] -> int8 NHWC, q = clamp(round((1/scale) * ((x / 255 - mean[c]) / std[c]))), every step one fp32
 * operation as in the torch pipeline.  mean3 / std3 are HOST pointers to three floats (copied at launch). */
int hawq_quantize_input_u8(hawq_handle* h, int32_t N, int32_t H, int32_t W, const uint8_t* x, const float* mean3,
                           const float* std3, float scale, int32_t lo, int32_t hi, int8_t* out, void* stream);

/* One image of a ragged batch: h x w x 3 uint8 pixels (HWC) at byte `offset` of the pixel arena.  h == 0: an absent slot. */
typedef struct {
  int64_t offset;
  int32_t h, w;
} hawq_image_desc;

/* The reference's evaluation transform (quant_train.py:427-438): Resize(S) -> CenterCrop(Ch, Cw) -> ToTensor -> Normalize ->
 * QuantAct input branch, for B images of any size in one launch.  table: DEVICE array of B hawq_image_desc into the DEVICE pixel
 * arena `pixels` of `pixel_bytes` bytes; out: int8 NHWC [B, Ch, Cw, 3].  The resize and crop are torchvision's on PIL images,
 * bit for bit (bilinear, 8 bits per channel); the last three steps are hawq_quantize_input_u8's table.  Every per-image quantity is
 * computed on the device, so the launch depends only on B, Ch and Cw (a captured graph serves any image sizes).  Requirements:
 * 256 <= S <= 16384, S >= max(Ch, Cw), 1 <= B <= 65535.  An entry with h == 0, a side outside 1..16384 or pixels outside the arena
 * is absent: its output is the quantised zero pixel.  mean3 / std3 are HOST pointers to three floats (copied at launch). */
int hawq_resize_crop_quantize_u8(hawq_handle* h, int32_t B, const uint8_t* pixels, int64_t pixel_bytes, const hawq_image_desc* table,
                                 int32_t S, int32_t Ch, int32_t Cw, const float* mean3, const float* std3, float scale, int32_t lo,
                                 int32_t hi, int8_t* out, void* stream);
/* fixedpoint_fn case 0 stand-alone (QuantAct after a conv or at unit entry): x [rows,C] (x_bits 16 = uint16 residual,
 * 32 = int32), per-channel chan (bias is added; pass 0) or scalar when chan_stride == 0 (chan[0] used for all).
 * Requires lo <= hi (else HAWQ_ERR_BAD_ARG, nothing launched) and C % 8 == 0 (else HAWQ_ERR_UNSUPPORTED). */
int hawq_requant(hawq_handle* h, int64_t rows, int32_t C, int32_t x_bits, const void* x, const hawq_chan* chan,
                 int32_t chan_stride, int32_t relu, int32_t out_bits, int32_t lo, int32_t hi, void* out, void* stream);
/* fixedpoint_fn case 1 stand-alone: y = [relu](RHE(res*m1/2^e1) + RHE((acc+bias)*m/2^e)); same operands as the fused form, checked
 * by the same rules as a RESIDUAL hawq_conv2d: res_kind 0 (res_bits 16 / 32, 1 <= res_e <= 62, res_m <= 2^31) or 1 (res_chan),
 * y_bits 0 / 16 / 32 (16 needs relu), low_bits 0 / 4 / 8 (the same range for low_m, low_e), at least one output; otherwise
 * HAWQ_ERR_BAD_ARG (nothing launched).  C % 8 != 0 returns HAWQ_ERR_UNSUPPORTED. */
int hawq_add_requant(hawq_handle* h, int64_t rows, int32_t C, const int32_t* acc, const hawq_chan* chan,
                     const hawq_epilogue_desc* ep, const void* res, const hawq_chan* res_chan,
                     void* y, void* out_low, void* stream);
/* integer tensor -> fp32 NCHW "fake-quant" value q * scale (graph edges of the module API). x_bits 4 (packed), 8, 16 (uint16), 32. */
int hawq_dequant_f32(hawq_handle* h, int32_t N, int32_t H, int32_t W, int32_t C, int32_t x_bits, int32_t x_signed,
                     const void* x, float scale, float* out_nchw, void* stream);
/* one value per byte (0..15) <-> packed nibbles in hawq nibble order; n_values % 8 == 0 */
int hawq_pack_i4(hawq_handle* h, int64_t n_values, const uint8_t* in, uint8_t* out, void* stream);
int hawq_unpack_i4(hawq_handle* h, int64_t n_values, const uint8_t* in, uint8_t* out, void* stream);

/* ---- host helpers (no GPU needed) --------------------------------------------------------------------------- */
/* batch_frexp (quant_utils.py:188-213) of one positive ratio: m = round_half_up(mant * 2^31), e = 31 - exp.
 * Returns HAWQ_ERR_UNSUPPORTED when e < 1 (ratio >= 2^30); for e > 62 the result is always 0: (m, e) := (0, 1). */
int hawq_dyadic(double ratio, uint32_t* m, int32_t* e);
/* exact host evaluation of RHE(v * m / 2^e) — the same routine the kernels inline */
int64_t hawq_rhe_requant_host(int32_t v, uint32_t m, int32_t e);
/* K permutation inside each 32-channel block for layers whose input is packed 4-bit (in place, int8 OHWI, host memory) */
int hawq_permute_weights_for_i4(int8_t* host_w, int64_t rows_times_taps, int32_t Cin);
/* Re-tile int8 OHWI weights [Cout][K]: block (n_tile, k_tile) = BN rows x 64 bytes (BN = 128 when Cout % 128 == 0, else 64),
 * stored contiguously with the shared-memory swizzle pre-applied (a k-tile of weights is one linear copy).  The convolution
 * kernels of this build read the OHWI part; hawq_conv2d_dual requires the layout.  `out` (Cout * K bytes) is normally w_ohwi + Cout * K, i.e. the copy is appended to the OHWI
 * tensor and announced with hawq_conv_desc.w_layout = 1.  Device pointers, asynchronous on the stream. */
int hawq_retile_weights(hawq_handle* h, const int8_t* w_ohwi, int32_t Cout, int64_t K, int8_t* out, void* stream);
/* debug: number of launches so far by kernel family: 0 = hawq_conv2d (wgmma implicit GEMM), 1 = hawq_dwconv3x3, 2 =
 * hawq_stem3x3_i8, 4 = hawq_conv2d_dual (both convolutions of a resize-unit tail in one kernel); 6 = hawq_stem_pool_i8 (fused
 * stem); families 3, 5 and 7 are unused in this build and stay 0;
 * -1 for an unknown family.  Lets tests assert which kernel ran. */
int64_t hawq_debug_kernel_count(int32_t family);
/* workspace query kept for ABI completeness: this build needs no scratch beyond caller tensors */
int64_t hawq_workspace_bytes(const hawq_conv_desc* d, const hawq_epilogue_desc* ep);

/* ---- engine files: a compiled forward saved to one file and replayed without Python (INTEGRATION.md §3) ------------ */
/* A plan file (CompiledModel.save) holds every launch of one forward as (entry id, arguments), for three sequences: "fast" (the
 * engine's residual stream width, ratio promises), "int32" (the fallback when the uint16 stream overflowed; absent when the fast
 * sequence already stores int32) and "safe" (no ratio promises: the fallback after HAWQ_FLAG_REQUANT_OVERFLOW).  Every pointer
 * argument is an offset into one of four regions: the input binding, the output binding (fp32 logits [N, classes], shared by the
 * three sequences), the constants (weights and per-channel tables, stored in the file) and the arena (every other buffer, laid out
 * with the aliasing of the recorded run; zeroed at load).  The loader captures each sequence into a CUDA graph that calls the entry
 * points of this header with exactly the recorded arguments, so a replay runs the same kernels on the same integers.
 *
 * Format (little-endian, fixed-width fields):
 *   header, 40 bytes: "HAWQPLAN", u32 format version (HAWQ_ENGINE_FORMAT), u32 HAWQ_ABI_VERSION, u32 compute capability major (9)
 *     and minor (0), u64 body bytes, u32 CRC-32 (zlib's) of the body, u32 zero;
 *   body: u32 input dtype (hawq_engine_dtype), u32 residual bits of the fast sequence (16 / 32), i64 input shape[4], i64 input bytes;
 *     i64 output shape[2]; u64 constant bytes, the constants; u64 arena bytes; u32 sequence count, then per sequence u32 kind
 *     (hawq_engine_seq), u32 record count, and per record u16 entry id (hawq_engine_entry), u16 argument count and the arguments
 *     in the entry's order without handle and stream, each a u8 kind (hawq_engine_arg) and its value: i32 / u32 / f32 4 bytes,
 *     i64 8 bytes, null nothing, ptr a u8 region (hawq_engine_region) and a u64 offset, blob a u32 length and the bytes (the value
 *     of a hawq_conv_desc, a hawq_epilogue_desc or a float[3] passed by pointer).
 * Trust: a plan file is trusted like a shared library.  Its structure is validated, its launches are not: the extents that a
 * descriptor determines are checked only by each entry point's own argument checks. */
#define HAWQ_ENGINE_FORMAT 1

/* entry ids of a plan file: the entry points a recorded forward launches */
enum hawq_engine_entry {
  HAWQ_ENTRY_CONV2D = 0,
  HAWQ_ENTRY_CONV2D_DUAL = 1,
  HAWQ_ENTRY_LINEAR_I8 = 2,
  HAWQ_ENTRY_STEM_CONV_I8 = 3,
  HAWQ_ENTRY_STEM_POOL_I8 = 4,
  HAWQ_ENTRY_DWCONV3X3 = 5,
  HAWQ_ENTRY_STEM3X3_I8 = 6,
  HAWQ_ENTRY_MAXPOOL_REQUANT = 7,
  HAWQ_ENTRY_AVGPOOL_REQUANT = 8,
  HAWQ_ENTRY_QUANTIZE_INPUT_F32 = 9,
  HAWQ_ENTRY_QUANTIZE_INPUT_U8 = 10,
  HAWQ_ENTRY_RESIZE_CROP_QUANTIZE_U8 = 11,
  HAWQ_ENTRY_REQUANT = 12,
  HAWQ_ENTRY_ADD_REQUANT = 13,
  HAWQ_ENTRY_DEQUANT_F32 = 14,
  HAWQ_ENTRY_PACK_I4 = 15,
  HAWQ_ENTRY_UNPACK_I4 = 16,
  HAWQ_ENTRY_COUNT = 17
};
enum hawq_engine_arg { HAWQ_ARG_I32 = 1, HAWQ_ARG_U32 = 2, HAWQ_ARG_I64 = 3, HAWQ_ARG_F32 = 4, HAWQ_ARG_NULL = 5, HAWQ_ARG_PTR = 6, HAWQ_ARG_BLOB = 7 };
enum hawq_engine_region { HAWQ_REGION_INPUT = 0, HAWQ_REGION_OUTPUT = 1, HAWQ_REGION_CONST = 2, HAWQ_REGION_ARENA = 3 };
enum hawq_engine_seq { HAWQ_SEQ_FAST = 0, HAWQ_SEQ_INT32 = 1, HAWQ_SEQ_SAFE = 2 };
/* input binding: int8 NHWC (already quantised), uint8 NHWC pixels, or fp32 NCHW (normalised) */
enum hawq_engine_dtype { HAWQ_DTYPE_INT8 = 0, HAWQ_DTYPE_UINT8 = 1, HAWQ_DTYPE_FLOAT32 = 2 };

typedef struct hawq_engine hawq_engine;

typedef struct {
  int32_t input_dtype;      /* hawq_engine_dtype */
  int32_t residual_bits;    /* of the fast sequence: 16 (an int32 sequence follows an overflow) or 32 */
  int64_t input_shape[4];
  int64_t input_bytes;
  int64_t output_shape[2];  /* fp32 [N, classes] */
  int64_t arena_bytes;
  int64_t constant_bytes;
  int64_t launches[3];      /* entry-point calls per sequence (hawq_engine_seq); 0: the sequence is absent */
  int64_t fallbacks;        /* a loaded engine: hawq_engine_run calls that replayed the int32 or safe sequence */
} hawq_engine_info;

/* Parses and validates a whole plan file in host memory without touching a device: magic, versions, checksum, every section and
 * record inside the buffer, entry ids and argument kinds and counts against each entry's signature, every ptr offset inside its
 * region.  HAWQ_ERR_BAD_ARG with a message on any failure; on success fills info (fallbacks 0) when info is not null. */
int hawq_engine_check(const void* data, int64_t bytes, hawq_engine_info* info);
/* Checks the file, creates the engine's own handle (its own status word) on `device`, allocates the regions, uploads the constants,
 * zeroes the arena and captures each sequence into a CUDA graph on a private stream.  The caller's current device is unchanged. */
int hawq_engine_load(int device, const void* data, int64_t bytes, hawq_engine** out);
/* frees everything the engine owns (synchronises its device) */
int hawq_engine_destroy(hawq_engine* eng);
/* device pointers of the input binding (input_bytes) and the output binding (fp32 [N, classes]) */
void* hawq_engine_input(const hawq_engine* eng);
float* hawq_engine_output(const hawq_engine* eng);
int hawq_engine_get_info(const hawq_engine* eng, hawq_engine_info* info);
/* resets the status word and replays the fast sequence on `stream`; the word is copied to a host-readable word at its end.  No host
 * synchronisation and no check: read the word with hawq_engine_status once the stream is synchronised */
int hawq_engine_enqueue(hawq_engine* eng, void* stream);
int hawq_engine_status(const hawq_engine* eng, int32_t* flags);
/* The exact forward: replays the fast sequence, synchronises `stream` and reads the status word (into *flags when not null).
 * HAWQ_FLAG_BAD_RATIO: returns HAWQ_ERR_RESULT_INVALID.  HAWQ_FLAG_REQUANT_OVERFLOW: replays the safe sequence.  Otherwise, with a
 * 16-bit fast sequence, HAWQ_FLAG_RESIDUAL_OVERFLOW replays the int32 sequence.  A fallback replay is enqueued on `stream` after
 * the fast one and counted in hawq_engine_info.fallbacks; the output binding holds the exact logits once `stream` reaches it. */
int hawq_engine_run(hawq_engine* eng, void* stream, int32_t* flags);

#ifdef __cplusplus
}
#endif
#endif /* HAWQ_B200_H */
