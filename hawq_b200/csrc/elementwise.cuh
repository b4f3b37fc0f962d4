// HBM-bound element-wise pieces of the HAWQ integer path: input quantisation, stand-alone case-0 / case-1
// requantisation (the unfused module API), average-pool tail, fp32 dequantisation, nibble (un)packing.
// All are one-pass, vectorised (8 channels per thread), grid-stride.
#pragma once
#include "common.cuh"

namespace hawq {

// load 8 consecutive channel values as int32 from a tensor of the given storage width
__device__ __forceinline__ void load8(const void* base, size_t idx, int bits, bool is_signed, int32_t (&v)[8]) {
  if (bits == 32) {
    const int4 a = *reinterpret_cast<const int4*>(reinterpret_cast<const int32_t*>(base) + idx);
    const int4 b = *reinterpret_cast<const int4*>(reinterpret_cast<const int32_t*>(base) + idx + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else if (bits == 16) {
    const uint4 a = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(base) + idx);
    const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (is_signed) {
        v[2 * k] = (int32_t)(int16_t)(w[k] & 0xFFFF);
        v[2 * k + 1] = (int32_t)(int16_t)(w[k] >> 16);
      } else {
        v[2 * k] = (int32_t)(w[k] & 0xFFFF);
        v[2 * k + 1] = (int32_t)(w[k] >> 16);
      }
    }
  } else if (bits == 8) {
    const uint2 a = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(base) + idx);
    const uint32_t w[2] = {a.x, a.y};
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint32_t b = (w[k >> 2] >> (8 * (k & 3))) & 0xFF;
      v[k] = is_signed ? (int32_t)(int8_t)b : (int32_t)b;
    }
  } else {  // 4: packed nibbles, hawq order (unsigned)
    const uint32_t a = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(base) + (idx >> 1));
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      v[k] = (int32_t)((a >> (8 * k)) & 0xF);
      v[k + 4] = (int32_t)((a >> (8 * k + 4)) & 0xF);
    }
  }
}

// store 8 consecutive channel values
__device__ __forceinline__ void store8(void* base, size_t idx, int bits, const int32_t (&v)[8]) {
  if (bits == 32) {
    int32_t* o = reinterpret_cast<int32_t*>(base) + idx;
    *reinterpret_cast<int4*>(o) = make_int4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<int4*>(o + 4) = make_int4(v[4], v[5], v[6], v[7]);
  } else if (bits == 16) {
    uint4 o;
    o.x = (uint32_t)(v[0] & 0xFFFF) | ((uint32_t)(v[1] & 0xFFFF) << 16);
    o.y = (uint32_t)(v[2] & 0xFFFF) | ((uint32_t)(v[3] & 0xFFFF) << 16);
    o.z = (uint32_t)(v[4] & 0xFFFF) | ((uint32_t)(v[5] & 0xFFFF) << 16);
    o.w = (uint32_t)(v[6] & 0xFFFF) | ((uint32_t)(v[7] & 0xFFFF) << 16);
    *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(base) + idx) = o;
  } else {
    uint32_t wlo = 0, whi = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      wlo |= (uint32_t)(v[k] & 0xFF) << (8 * k);
      whi |= (uint32_t)(v[k + 4] & 0xFF) << (8 * k);
    }
    if (bits == 8) *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(base) + idx) = make_uint2(wlo, whi);
    else *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(base) + (idx >> 1)) = pack_nibbles8(wlo, whi);
  }
}

// QuantAct input branch: q = clamp(rint((1/scale) * x)); fp32 NCHW -> int8 NHWC.  One thread per pixel.
__global__ void __launch_bounds__(256) quantize_input_kernel(const float* __restrict__ x, int N, int C, int H, int W,
                                                             float inv_scale, int lo, int hi, int8_t* __restrict__ out) {
  const long long hw = (long long)H * W, total = (long long)N * hw;
  for (long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x; id < total;
       id += (long long)gridDim.x * blockDim.x) {
    const long long n = id / hw, pix = id - n * hw;
    for (int c = 0; c < C; ++c) {
      const float v = rintf(__fmul_rn(inv_scale, x[(n * C + c) * hw + pix]));
      const int q = (int)fminf(fmaxf(v, (float)lo), (float)hi);
      out[id * C + c] = (int8_t)q;
    }
  }
}

// uint8 pixel -> int8 network input table of the uint8 image pipelines (SURVEY.md 8(f) rank 2;
// tvm_benchmark/test_resnet_accuracy_imagenet.py:62-75,82-93): ToTensor (u / 255), Normalize ((v - mean_c) / std_c) and the QuantAct
// input branch (clamp(rint((1/scale) * x))).  Every step is the same single fp32 operation the reference's torch pipeline performs,
// so the integers are identical; with 256 possible inputs per channel the whole map is a 3 x 256 table, lut[c << 8 | u], built by
// the calling block in shared memory (the caller synchronises before reading it).
__device__ __forceinline__ void build_input_lut(int8_t* lut, float m0, float m1, float m2, float s0, float s1, float s2, float inv_scale,
                                                int lo, int hi) {
  for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) {
    const int c = i >> 8, u = i & 255;
    const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
    const float v = __fdiv_rn(__fsub_rn(__fdiv_rn((float)u, 255.0f), mean), sd);
    const float q = rintf(__fmul_rn(inv_scale, v));
    lut[i] = (int8_t)(int)fminf(fmaxf(q, (float)lo), (float)hi);
  }
}

// uint8 NHWC -> int8 NHWC through the build_input_lut table, one pass.
__global__ void __launch_bounds__(256) quantize_input_u8_kernel(const uint8_t* __restrict__ x, long long n_bytes, int C,
                                                                float m0, float m1, float m2, float s0, float s1, float s2,
                                                                float inv_scale, int lo, int hi, int8_t* __restrict__ out) {
  __shared__ int8_t lut[3 * 256];
  build_input_lut(lut, m0, m1, m2, s0, s1, s2, inv_scale, lo, hi);
  __syncthreads();
  const long long words = n_bytes >> 2;
  for (long long wi = blockIdx.x * (long long)blockDim.x + threadIdx.x; wi < words; wi += (long long)gridDim.x * blockDim.x) {
    const uint32_t v = reinterpret_cast<const uint32_t*>(x)[wi];
    int c = (int)((wi * 4) % C);
    uint32_t o = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      o |= (uint32_t)(uint8_t)lut[(c << 8) | ((v >> (8 * j)) & 0xFF)] << (8 * j);
      c = (c + 1 == C) ? 0 : c + 1;
    }
    reinterpret_cast<uint32_t*>(out)[wi] = o;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n_bytes & 3)) {          // tail bytes
    const long long i = (words << 2) + threadIdx.x;
    out[i] = lut[((int)(i % C) << 8) | x[i]];
  }
}

// case 0 stand-alone: out = clamp(RHE(([relu](x + bias)) * m / 2^e)).
__global__ void __launch_bounds__(256) requant_kernel(const void* __restrict__ x, long long rows, int C, int x_bits,
                                                      const hawq_chan* __restrict__ chan, int chan_stride, int relu,
                                                      int out_bits, int lo, int hi, void* __restrict__ out) {
  const int c8 = C / 8;
  const long long total = rows * c8;
  for (long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x; id < total;
       id += (long long)gridDim.x * blockDim.x) {
    const int cg = (int)(id % c8);
    const size_t idx = (size_t)(id / c8) * C + cg * 8;
    int32_t v[8], q[8];
    load8(x, idx, x_bits, false, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const hawq_chan ch = chan[(size_t)(cg * 8 + k) * chan_stride];
      int32_t a = sat_add(v[k], ch.bias);
      if (relu) a = max(a, 0);
      q[k] = clampi(rhe_requant(a, ch.m, ch.e), lo, hi);
    }
    store8(out, idx, out_bits, q);
  }
}

// case 1 stand-alone.
struct AddRequantParams {
  const int32_t* acc;
  const hawq_chan* chan;
  const void* res;
  const hawq_chan* res_chan;
  void* y;
  void* out_low;
  int32_t* status;
  long long rows;
  int C, relu, res_kind, res_bits;
  uint32_t res_m;
  int res_e, y_bits, low_bits;
  uint32_t low_m;
  int low_e, low_lo, low_hi;
};

__global__ void __launch_bounds__(256) add_requant_kernel(const AddRequantParams p) {
  const int c8 = p.C / 8;
  const long long total = p.rows * c8;
  for (long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x; id < total;
       id += (long long)gridDim.x * blockDim.x) {
    const int cg = (int)(id % c8);
    const size_t idx = (size_t)(id / c8) * p.C + cg * 8;
    int32_t a[8], r[8], y[8], q[8];
    load8(p.acc, idx, 32, true, a);
    load8(p.res, idx, p.res_kind == 1 ? 32 : p.res_bits, false, r);
    bool over = false;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = cg * 8 + k;
      const hawq_chan ch = p.chan[c];
      uint32_t rm = p.res_m;
      int re = p.res_e;
      if (p.res_kind == 1) { rm = p.res_chan[c].m; re = p.res_chan[c].e; }
      int32_t s = sat_add(rhe_requant(r[k], rm, re), rhe_requant(sat_add(a[k], ch.bias), ch.m, ch.e));
      if (p.relu) s = max(s, 0);
      y[k] = s;
      if (p.low_bits) q[k] = clampi(rhe_requant(s, p.low_m, p.low_e), p.low_lo, p.low_hi);
    }
    if (p.y_bits == 16) {
#pragma unroll
      for (int k = 0; k < 8; ++k) { over |= y[k] > 65535; y[k] = min(y[k], 65535); }
      if (over) atomicOr(p.status, HAWQ_FLAG_RESIDUAL_OVERFLOW);
    }
    if (p.y_bits) store8(p.y, idx, p.y_bits, y);
    if (p.low_bits) store8(p.out_low, idx, p.low_bits, q);
  }
}

// QuantAveragePool2d + quant_act_output: x [N, HW, C] residual stream -> int8 [N, C].  One thread per (n, c).
__global__ void __launch_bounds__(256) avgpool_requant_kernel(const void* __restrict__ x, int N, int HW, int C,
                                                              int x_bits, uint32_t m, int e, int lo, int hi,
                                                              int8_t* __restrict__ out) {
  const long long total = (long long)N * C;
  for (long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x; id < total;
       id += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(id % C);
    const long long n = id / C;
    long long s = 0;
    for (int k = 0; k < HW; ++k) {
      const size_t idx = ((size_t)n * HW + k) * C + c;
      s += (x_bits == 16) ? (long long)reinterpret_cast<const uint16_t*>(x)[idx]
                          : (long long)reinterpret_cast<const int32_t*>(x)[idx];
    }
    out[id] = (int8_t)clampi(rhe_requant(trunc_avg(s, HW), m, e), lo, hi);
  }
}

// QuantLinear tail (quant_modules.py:79-130): out[n][c] = float(sat32(x[n,:] . w[c,:] + bias[c])) * fscale[c].
// A batch-rows x K x 1000 GEMM is too small for 128 x 128 tensor-core tiles (8 CTAs on 148 SMs), so this kernel spreads
// the channels over the chip instead: one CTA per 8 output channels (their weights sit in shared memory and are read as
// warp-wide broadcasts), one thread per (row, 4-channel group), x staged through shared memory in 128-byte slabs
// (coalesced cp.async, double buffered, rows padded to 144 B so that row-per-lane 16-byte reads are conflict-free), dp4a.
constexpr int LIN_CH = 8, LIN_ROWS = 128, LIN_SLAB = 128, LIN_PITCH = LIN_SLAB + 16;
constexpr int LIN_MAX_K = 8192;
inline int linear_smem_bytes(int K) { return LIN_CH * K + 2 * LIN_ROWS * LIN_PITCH; }

__global__ void __launch_bounds__(256) linear_dp4a_kernel(const int8_t* __restrict__ x, const int8_t* __restrict__ w,
                                                          const hawq_chan* __restrict__ chan, const float* __restrict__ fscale,
                                                          float* __restrict__ out, int N, int K, int Cout) {
  extern __shared__ __align__(16) uint8_t lin_smem[];
  uint8_t* sW = lin_smem;                       // [LIN_CH][K]
  uint8_t* sX = lin_smem + LIN_CH * K;          // [2][LIN_ROWS][LIN_PITCH]
  const int tid = threadIdx.x;
  const int c0 = blockIdx.x * LIN_CH;
  const int row0 = blockIdx.y * LIN_ROWS;
  const int row = tid & (LIN_ROWS - 1), cg = tid >> 7;     // a warp shares cg: weight reads are broadcasts
  const int slabs = K / LIN_SLAB;

  auto load_slab = [&](int s, int buf) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int id = tid + i * 256;
      const int r = id >> 3, col = id & 7;
      const bool v = row0 + r < N;
      const int8_t* src = v ? x + (size_t)(row0 + r) * K + s * LIN_SLAB + col * 16 : x;
      cp_async_16((uint32_t)__cvta_generic_to_shared(sX + (buf * LIN_ROWS + r) * LIN_PITCH + col * 16), src, v ? 16 : 0);
    }
    cp_async_commit();
  };
  load_slab(0, 0);
  for (int i = tid; i < LIN_CH * K / 16; i += 256)        // the 8 weight rows are contiguous in global memory
    reinterpret_cast<int4*>(sW)[i] = reinterpret_cast<const int4*>(w + (size_t)c0 * K)[i];

  int acc[4] = {0, 0, 0, 0};
  for (int s = 0; s < slabs; ++s) {
    if (s + 1 < slabs) { load_slab(s + 1, (s + 1) & 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncthreads();
    const uint8_t* xr = sX + ((s & 1) * LIN_ROWS + row) * LIN_PITCH;
#pragma unroll
    for (int col = 0; col < 8; ++col) {
      const int4 xv = *reinterpret_cast<const int4*>(xr + col * 16);
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) {
        const int4 wv = *reinterpret_cast<const int4*>(sW + (size_t)(cg * 4 + ch) * K + s * LIN_SLAB + col * 16);
        acc[ch] = __dp4a(xv.x, wv.x, acc[ch]);
        acc[ch] = __dp4a(xv.y, wv.y, acc[ch]);
        acc[ch] = __dp4a(xv.z, wv.z, acc[ch]);
        acc[ch] = __dp4a(xv.w, wv.w, acc[ch]);
      }
    }
    __syncthreads();                                       // the buffer is refilled two iterations later
  }
  if (row0 + row < N) {
#pragma unroll
    for (int ch = 0; ch < 4; ++ch) {
      const int c = c0 + cg * 4 + ch;
      if (c < Cout) out[(size_t)(row0 + row) * Cout + c] = __int2float_rn(sat_add(acc[ch], chan[c].bias)) * fscale[c];
    }
  }
}

// integer NHWC -> fp32 NCHW value q * scale (fp32 multiply, as quant_modules.py:303).  One thread per output element.
__global__ void __launch_bounds__(256) dequant_f32_kernel(const void* __restrict__ x, int N, int H, int W, int C,
                                                          int x_bits, int x_signed, float scale,
                                                          float* __restrict__ out) {
  const long long hw = (long long)H * W, total = (long long)N * C * hw;
  for (long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x; id < total;
       id += (long long)gridDim.x * blockDim.x) {
    const long long pix = id % hw;
    const int c = (int)((id / hw) % C);
    const long long n = id / (hw * C);
    const size_t idx = ((size_t)n * hw + pix) * C + c;
    int32_t q;
    if (x_bits == 32) q = reinterpret_cast<const int32_t*>(x)[idx];
    else if (x_bits == 16) q = x_signed ? (int32_t)reinterpret_cast<const int16_t*>(x)[idx]
                                        : (int32_t)reinterpret_cast<const uint16_t*>(x)[idx];
    else if (x_bits == 8) q = x_signed ? (int32_t)reinterpret_cast<const int8_t*>(x)[idx]
                                       : (int32_t)reinterpret_cast<const uint8_t*>(x)[idx];
    else {
      const size_t grp = idx >> 3;
      const int k = (int)(idx & 7);
      const uint8_t b = reinterpret_cast<const uint8_t*>(x)[grp * 4 + (k & 3)];
      q = (k < 4) ? (b & 0xF) : (b >> 4);
    }
    out[id] = __fmul_rn((float)q, scale);
  }
}

__global__ void __launch_bounds__(256) pack_i4_kernel(const uint8_t* __restrict__ in, long long n8,
                                                      uint8_t* __restrict__ out) {
  for (long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x; id < n8;
       id += (long long)gridDim.x * blockDim.x) {
    const uint2 a = *reinterpret_cast<const uint2*>(in + id * 8);
    *reinterpret_cast<uint32_t*>(out + id * 4) = pack_nibbles8(a.x, a.y);
  }
}

__global__ void __launch_bounds__(256) unpack_i4_kernel(const uint8_t* __restrict__ in, long long n8,
                                                        uint8_t* __restrict__ out) {
  for (long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x; id < n8;
       id += (long long)gridDim.x * blockDim.x) {
    const uint32_t a = *reinterpret_cast<const uint32_t*>(in + id * 4);
    *reinterpret_cast<uint2*>(out + id * 8) = make_uint2(a & 0x0F0F0F0Fu, (a >> 4) & 0x0F0F0F0Fu);
  }
}

// One-time re-tiling of OHWI int8 weights (hawq_conv2d_desc.w_layout 1): block (n_tile, k_tile) = BN rows x 64 bytes, stored
// contiguously with the SWIZZLE_64B pattern already applied (the shared-memory B tile of conv_igemm.cuh).
__global__ void __launch_bounds__(256) retile_weights_kernel(const int8_t* __restrict__ w, int Cout, int K, int BN, int8_t* __restrict__ out) {
  const int kt_total = K / 64;
  const long long chunks = (long long)Cout * K / 16;
  for (long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x; id < chunks; id += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(id & 3);
    const long long rk = id >> 2;                 // (row, k-tile)
    const int kt = (int)(rk % kt_total);
    const int row = (int)(rk / kt_total);
    const int nt = row / BN, r = row % BN;
    const int4 v = *reinterpret_cast<const int4*>(w + (size_t)row * K + kt * 64 + c * 16);
    *reinterpret_cast<int4*>(out + ((size_t)nt * kt_total + kt) * BN * 64 + r * 64 + ((c ^ ((r >> 1) & 3)) << 4)) = v;
  }
}

}  // namespace hawq
