// Engine files (include/hawq_b200.h, INTEGRATION.md §3): the device-free checker of a plan file and the runtime that captures its
// sequences into CUDA graphs by calling this library's own entry points with the recorded arguments.  Host code only: no kernel.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/hawq_b200.h"

namespace hawq {
int fail(int code, const char* fmt, ...);   // api.cu: the thread's hawq_last_error message
}
using hawq::fail;

namespace {

constexpr char kMagic[8] = {'H', 'A', 'W', 'Q', 'P', 'L', 'A', 'N'};
constexpr size_t kHeaderBytes = 40;
constexpr int64_t kMaxRegion = 1ll << 40;      // no region of a plan file comes near a terabyte
constexpr uint32_t kMaxRecords = 1u << 20;

// Arguments of each entry (hawq_engine_entry order) without handle and stream: i int32, u uint32, I int64, f float, p pointer (ptr or
// null), D hawq_conv_desc, E hawq_epilogue_desc, F float[3] (the three by value).  hawq_b200/engine_file.py (arg_codes) derives the
// same strings from the ctypes signatures of hawq_b200/_lib.py; tests/test_engine_file_cpu.py keeps the two equal.
const char* const kEntryArgs[HAWQ_ENTRY_COUNT] = {
    "DEpppppppp",        // hawq_conv2d
    "DEpppDppppp",       // hawq_conv2d_dual
    "iiiippppp",         // hawq_linear_i8
    "iiipppiip",         // hawq_stem_conv_i8
    "iiipppiiipiuiiip",  // hawq_stem_pool_i8
    "iiiiiipppiiiip",    // hawq_dwconv3x3
    "iiipppiiiipiuiiip", // hawq_stem3x3_i8
    "iiiipipiuiiip",     // hawq_maxpool_requant
    "iiiipuiiip",        // hawq_avgpool_requant
    "iiiipfiip",         // hawq_quantize_input_f32
    "iiipFFfiip",        // hawq_quantize_input_u8
    "ipIpiiiFFfiip",     // hawq_resize_crop_quantize_u8
    "Iiippiiiiip",       // hawq_requant
    "IippEpppp",         // hawq_add_requant
    "iiiiiipfp",         // hawq_dequant_f32
    "Ipp",               // hawq_pack_i4
    "Ipp",               // hawq_unpack_i4
};

struct Arg {
  uint8_t kind;
  uint8_t region;
  int64_t i;          // I32 / I64 value, PTR offset
  uint32_t u;
  float f;
  const uint8_t* blob;
};

struct Record {
  uint16_t entry;
  std::vector<Arg> args;
};

struct Plan {
  hawq_engine_info info;
  const uint8_t* constants;
  bool present[3];
  std::vector<Record> seq[3];
};

uint32_t crc32(const uint8_t* p, size_t n) {   // zlib's CRC-32 (reflected polynomial 0xEDB88320)
  static uint32_t table[256];
  static bool ready = [] {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
      table[i] = c;
    }
    return true;
  }();
  (void)ready;
  uint32_t c = 0xFFFFFFFFu;
  for (size_t i = 0; i < n; ++i) c = table[(c ^ p[i]) & 0xFF] ^ (c >> 8);
  return c ^ 0xFFFFFFFFu;
}

// Bounds-checked little-endian reader over the file; any read past the end leaves ok false
struct Reader {
  const uint8_t* p;
  size_t n, pos;
  bool ok;
  const uint8_t* take(size_t k) {
    if (!ok || n - pos < k) { ok = false; return nullptr; }
    const uint8_t* r = p + pos;
    pos += k;
    return r;
  }
  template <class T> T get() {
    T v{};
    if (const uint8_t* r = take(sizeof(T))) memcpy(&v, r, sizeof(T));
    return v;
  }
};

size_t blob_bytes(char code) { return code == 'D' ? sizeof(hawq_conv_desc) : code == 'E' ? sizeof(hawq_epilogue_desc) : 3 * sizeof(float); }

int bad(const char* fmt, long long a = 0, long long b = 0, long long c = 0) {
  char msg[256];
  snprintf(msg, sizeof(msg), fmt, a, b, c);
  return fail(HAWQ_ERR_BAD_ARG, "hawq_engine_check: %s", msg);
}

int parse(const void* data, int64_t bytes, Plan* plan) {
  if (!data || bytes < (int64_t)kHeaderBytes) return bad("no data or %lld bytes, shorter than the header", bytes);
  const uint8_t* p = (const uint8_t*)data;
  Reader h{p, kHeaderBytes, 0, true};
  if (memcmp(h.take(8), kMagic, 8) != 0) return bad("not a plan file (magic)");
  const uint32_t format = h.get<uint32_t>(), abi = h.get<uint32_t>(), cc_major = h.get<uint32_t>(), cc_minor = h.get<uint32_t>();
  const uint64_t body_bytes = h.get<uint64_t>();
  const uint32_t crc = h.get<uint32_t>(), zero = h.get<uint32_t>();
  if (format != HAWQ_ENGINE_FORMAT) return bad("format version %lld, this library reads %lld", format, HAWQ_ENGINE_FORMAT);
  if (abi != HAWQ_ABI_VERSION) return bad("ABI version %lld, this library has %lld", abi, HAWQ_ABI_VERSION);
  if (cc_major != 9 || cc_minor != 0) return bad("made for compute capability %lld.%lld, this library runs 9.0", cc_major, cc_minor);
  if (zero != 0) return bad("reserved header field is not zero");
  if (body_bytes != (uint64_t)bytes - kHeaderBytes) return bad("body of %lld bytes declared, %lld present", (long long)body_bytes, bytes - (long long)kHeaderBytes);
  const uint8_t* body = p + kHeaderBytes;
  if (crc32(body, body_bytes) != crc) return bad("checksum mismatch");

  Reader r{body, (size_t)body_bytes, 0, true};
  hawq_engine_info& in = plan->info;
  memset(&in, 0, sizeof(in));
  in.input_dtype = r.get<int32_t>();
  in.residual_bits = r.get<int32_t>();
  for (int i = 0; i < 4; ++i) in.input_shape[i] = r.get<int64_t>();
  in.input_bytes = r.get<int64_t>();
  for (int i = 0; i < 2; ++i) in.output_shape[i] = r.get<int64_t>();
  if (!r.ok) return bad("truncated bindings");
  if (in.input_dtype < HAWQ_DTYPE_INT8 || in.input_dtype > HAWQ_DTYPE_FLOAT32) return bad("unknown input dtype %lld", in.input_dtype);
  if (in.residual_bits != 16 && in.residual_bits != 32) return bad("residual bits %lld (16 or 32)", in.residual_bits);
  long long elems = 1;
  for (int i = 0; i < 4; ++i) {
    if (in.input_shape[i] < 1 || in.input_shape[i] > (1ll << 31)) return bad("input extent %lld out of range", in.input_shape[i]);
    elems *= in.input_shape[i];
    if (elems > kMaxRegion) return bad("input too large");
  }
  if (in.input_bytes != elems * (in.input_dtype == HAWQ_DTYPE_FLOAT32 ? 4 : 1)) return bad("input of %lld bytes for its shape", in.input_bytes);
  if (in.output_shape[0] < 1 || in.output_shape[1] < 1 || in.output_shape[0] > (1ll << 20) || in.output_shape[1] > (1ll << 20))
    return bad("output shape %lld x %lld out of range", in.output_shape[0], in.output_shape[1]);
  const uint64_t const_bytes = r.get<uint64_t>();
  if (!r.ok || const_bytes > r.n - r.pos) return bad("constants of %lld bytes run past the file", (long long)const_bytes);
  in.constant_bytes = (int64_t)const_bytes;
  plan->constants = r.take(const_bytes);
  const uint64_t arena_bytes = r.get<uint64_t>();
  if (!r.ok || arena_bytes > (uint64_t)kMaxRegion) return bad("arena of %lld bytes out of range", (long long)arena_bytes);
  in.arena_bytes = (int64_t)arena_bytes;
  const int64_t region_bytes[4] = {in.input_bytes, in.output_shape[0] * in.output_shape[1] * 4, in.constant_bytes, in.arena_bytes};

  const uint32_t n_seq = r.get<uint32_t>();
  if (!r.ok || n_seq < 2 || n_seq > 3) return bad("%lld sequences (2 or 3)", n_seq);
  for (int k = 0; k < 3; ++k) plan->present[k] = false;
  for (uint32_t s = 0; s < n_seq; ++s) {
    const uint32_t kind = r.get<uint32_t>(), n_rec = r.get<uint32_t>();
    if (!r.ok) return bad("truncated sequence header");
    if (kind > HAWQ_SEQ_SAFE || plan->present[kind]) return bad("sequence kind %lld unknown or repeated", kind);
    if (n_rec < 1 || n_rec > kMaxRecords) return bad("sequence %lld has %lld records", kind, n_rec);
    plan->present[kind] = true;
    std::vector<Record>& recs = plan->seq[kind];
    recs.clear();   // grown record by record: a count the file cannot back is caught as a truncation, not allocated
    for (uint32_t j = 0; j < n_rec; ++j) {
      recs.emplace_back();
      Record& rec = recs.back();
      rec.entry = r.get<uint16_t>();
      const uint16_t n_args = r.get<uint16_t>();
      if (!r.ok) return bad("sequence %lld record %lld truncated", kind, j);
      if (rec.entry >= HAWQ_ENTRY_COUNT) return bad("sequence %lld record %lld: unknown entry id %lld", kind, j, rec.entry);
      const char* sig = kEntryArgs[rec.entry];
      if (n_args != strlen(sig)) return bad("record %lld: entry %lld takes %lld arguments", j, rec.entry, (long long)strlen(sig));
      rec.args.resize(n_args);
      for (uint16_t a = 0; a < n_args; ++a) {
        Arg& x = rec.args[a];
        memset(&x, 0, sizeof(x));
        x.kind = r.get<uint8_t>();
        const char code = sig[a];
        const int want = code == 'i' ? HAWQ_ARG_I32 : code == 'u' ? HAWQ_ARG_U32 : code == 'I' ? HAWQ_ARG_I64 : code == 'f' ? HAWQ_ARG_F32
                         : code == 'p' ? HAWQ_ARG_PTR : HAWQ_ARG_BLOB;
        if (!(x.kind == want || (code == 'p' && x.kind == HAWQ_ARG_NULL)))
          return bad("record %lld argument %lld: kind %lld does not match the entry's signature", j, a, x.kind);
        switch (x.kind) {
          case HAWQ_ARG_I32: x.i = r.get<int32_t>(); break;
          case HAWQ_ARG_U32: x.u = r.get<uint32_t>(); break;
          case HAWQ_ARG_I64: x.i = r.get<int64_t>(); break;
          case HAWQ_ARG_F32: x.f = r.get<float>(); break;
          case HAWQ_ARG_NULL: break;
          case HAWQ_ARG_PTR: {
            x.region = r.get<uint8_t>();
            const uint64_t off = r.get<uint64_t>();
            if (!r.ok) break;
            if (x.region > HAWQ_REGION_ARENA || off >= (uint64_t)region_bytes[x.region])
              return bad("record %lld argument %lld: pointer outside its region (region %lld)", j, a, x.region);
            x.i = (int64_t)off;
            break;
          }
          default: {   // HAWQ_ARG_BLOB
            const uint32_t len = r.get<uint32_t>();
            if (r.ok && len != blob_bytes(code)) return bad("record %lld argument %lld: blob of %lld bytes", j, a, len);
            x.blob = r.take(len);
          }
        }
        if (!r.ok) return bad("record %lld argument %lld truncated", j, a);
      }
    }
    in.launches[kind] = n_rec;
  }
  if (!plan->present[HAWQ_SEQ_FAST] || !plan->present[HAWQ_SEQ_SAFE] || plan->present[HAWQ_SEQ_INT32] != (in.residual_bits == 16))
    return bad("sequences fast and safe, and int32 exactly when the fast sequence is 16-bit, are required");
  if (r.pos != r.n) return bad("%lld bytes after the last sequence", (long long)(r.n - r.pos));
  return HAWQ_OK;
}

// One call of the recorded entry point with the record's arguments (pointers rebased on the engine's regions)
int call(hawq_handle* h, const Record& rec, void* const* base, cudaStream_t s) {
  const std::vector<Arg>& a = rec.args;
  auto P = [&](int k) -> void* { return a[k].kind == HAWQ_ARG_PTR ? (char*)base[a[k].region] + a[k].i : nullptr; };
  auto I = [&](int k) { return (int32_t)a[k].i; };
  auto L = [&](int k) { return (int64_t)a[k].i; };
  auto U = [&](int k) { return a[k].u; };
  auto F = [&](int k) { return a[k].f; };
  hawq_conv_desc d, d2;
  hawq_epilogue_desc ep;
  float f3[2][3];
  auto B = [&](int k, void* dst, size_t n) { memcpy(dst, a[k].blob, n); };
  using c8 = const int8_t;
  using ch = const hawq_chan;
  switch (rec.entry) {
    case HAWQ_ENTRY_CONV2D:
      B(0, &d, sizeof d); B(1, &ep, sizeof ep);
      return hawq_conv2d(h, &d, &ep, P(2), (c8*)P(3), (ch*)P(4), P(5), (ch*)P(6), (const float*)P(7), P(8), P(9), s);
    case HAWQ_ENTRY_CONV2D_DUAL:
      B(0, &d, sizeof d); B(1, &ep, sizeof ep); B(5, &d2, sizeof d2);
      return hawq_conv2d_dual(h, &d, &ep, P(2), (c8*)P(3), (ch*)P(4), &d2, P(6), (c8*)P(7), (ch*)P(8), P(9), P(10), s);
    case HAWQ_ENTRY_LINEAR_I8:
      return hawq_linear_i8(h, I(0), I(1), I(2), I(3), (c8*)P(4), (c8*)P(5), (ch*)P(6), (const float*)P(7), (float*)P(8), s);
    case HAWQ_ENTRY_STEM_CONV_I8:
      return hawq_stem_conv_i8(h, I(0), I(1), I(2), (c8*)P(3), (c8*)P(4), (ch*)P(5), I(6), I(7), (int16_t*)P(8), s);
    case HAWQ_ENTRY_STEM_POOL_I8:
      return hawq_stem_pool_i8(h, I(0), I(1), I(2), (c8*)P(3), (c8*)P(4), (ch*)P(5), I(6), I(7), I(8), P(9), I(10), U(11), I(12), I(13),
                               I(14), P(15), s);
    case HAWQ_ENTRY_DWCONV3X3:
      return hawq_dwconv3x3(h, I(0), I(1), I(2), I(3), I(4), I(5), P(6), (c8*)P(7), (ch*)P(8), I(9), I(10), I(11), I(12), P(13), s);
    case HAWQ_ENTRY_STEM3X3_I8:
      return hawq_stem3x3_i8(h, I(0), I(1), I(2), (c8*)P(3), (c8*)P(4), (ch*)P(5), I(6), I(7), I(8), I(9), P(10), I(11), U(12), I(13),
                             I(14), I(15), P(16), s);
    case HAWQ_ENTRY_MAXPOOL_REQUANT:
      return hawq_maxpool_requant(h, I(0), I(1), I(2), I(3), (const int16_t*)P(4), I(5), P(6), I(7), U(8), I(9), I(10), I(11), P(12), s);
    case HAWQ_ENTRY_AVGPOOL_REQUANT:
      return hawq_avgpool_requant(h, I(0), I(1), I(2), I(3), P(4), U(5), I(6), I(7), I(8), (int8_t*)P(9), s);
    case HAWQ_ENTRY_QUANTIZE_INPUT_F32:
      return hawq_quantize_input_f32(h, I(0), I(1), I(2), I(3), (const float*)P(4), F(5), I(6), I(7), (int8_t*)P(8), s);
    case HAWQ_ENTRY_QUANTIZE_INPUT_U8:
      B(4, f3[0], sizeof f3[0]); B(5, f3[1], sizeof f3[1]);
      return hawq_quantize_input_u8(h, I(0), I(1), I(2), (const uint8_t*)P(3), f3[0], f3[1], F(6), I(7), I(8), (int8_t*)P(9), s);
    case HAWQ_ENTRY_RESIZE_CROP_QUANTIZE_U8:
      B(7, f3[0], sizeof f3[0]); B(8, f3[1], sizeof f3[1]);
      return hawq_resize_crop_quantize_u8(h, I(0), (const uint8_t*)P(1), L(2), (const hawq_image_desc*)P(3), I(4), I(5), I(6), f3[0],
                                          f3[1], F(9), I(10), I(11), (int8_t*)P(12), s);
    case HAWQ_ENTRY_REQUANT:
      return hawq_requant(h, L(0), I(1), I(2), P(3), (ch*)P(4), I(5), I(6), I(7), I(8), I(9), P(10), s);
    case HAWQ_ENTRY_ADD_REQUANT:
      B(4, &ep, sizeof ep);
      return hawq_add_requant(h, L(0), I(1), (const int32_t*)P(2), (ch*)P(3), &ep, P(5), (ch*)P(6), P(7), P(8), s);
    case HAWQ_ENTRY_DEQUANT_F32:
      return hawq_dequant_f32(h, I(0), I(1), I(2), I(3), I(4), I(5), P(6), F(7), (float*)P(8), s);
    case HAWQ_ENTRY_PACK_I4:
      return hawq_pack_i4(h, L(0), (const uint8_t*)P(1), (uint8_t*)P(2), s);
    case HAWQ_ENTRY_UNPACK_I4:
      return hawq_unpack_i4(h, L(0), (const uint8_t*)P(1), (uint8_t*)P(2), s);
  }
  return fail(HAWQ_ERR_BAD_ARG, "hawq_engine: unknown entry id %d", rec.entry);
}

}  // namespace

struct hawq_engine {
  int device;
  hawq_handle* h;
  cudaStream_t stream;         // private capture stream
  void* region[4];             // hawq_engine_region
  int32_t* status_copy;        // device word the graphs copy the handle's status word into
  int32_t* host_status;        // pinned host word the graphs copy it on to
  cudaGraph_t graph[3];
  cudaGraphExec_t exec[3];
  hawq_engine_info info;
};

#define ENG_TRY(expr)                                                                                          \
  do {                                                                                                         \
    cudaError_t _e = (expr);                                                                                   \
    if (_e != cudaSuccess) return fail(HAWQ_ERR_CUDA, "hawq_engine: %s: %s", #expr, cudaGetErrorString(_e));   \
  } while (0)

namespace {

// Captures sequence k: reset the status word, every record, copy the word to the host-readable word
int capture(hawq_engine* e, const std::vector<Record>& recs, int k) {
  ENG_TRY(cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal));
  int rc = hawq_reset_status(e->h, e->stream);
  for (size_t j = 0; rc == HAWQ_OK && j < recs.size(); ++j) rc = call(e->h, recs[j], e->region, e->stream);
  if (rc == HAWQ_OK) rc = hawq_copy_status(e->h, e->status_copy, e->stream);
  if (rc == HAWQ_OK && cudaMemcpyAsync(e->host_status, e->status_copy, sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream) != cudaSuccess)
    rc = fail(HAWQ_ERR_CUDA, "hawq_engine_load: status copy: %s", cudaGetErrorString(cudaGetLastError()));
  cudaGraph_t g = nullptr;
  const cudaError_t end = cudaStreamEndCapture(e->stream, &g);
  if (rc != HAWQ_OK) {
    if (g) cudaGraphDestroy(g);
    return rc;
  }
  if (end != cudaSuccess) return fail(HAWQ_ERR_CUDA, "hawq_engine_load: capture of sequence %d: %s", k, cudaGetErrorString(end));
  e->graph[k] = g;
  ENG_TRY(cudaGraphInstantiate(&e->exec[k], g, 0));
  return HAWQ_OK;
}

int load_on(int device, const Plan& plan, hawq_engine* e) {
  ENG_TRY(cudaSetDevice(device));
  if (int rc = hawq_create(device, &e->h)) return rc;
  ENG_TRY(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
  const int64_t bytes[4] = {e->info.input_bytes, e->info.output_shape[0] * e->info.output_shape[1] * 4, e->info.constant_bytes,
                            e->info.arena_bytes};
  for (int k = 0; k < 4; ++k) {
    ENG_TRY(cudaMalloc(&e->region[k], bytes[k] > 0 ? (size_t)bytes[k] : 16));
    ENG_TRY(cudaMemset(e->region[k], 0, bytes[k] > 0 ? (size_t)bytes[k] : 16));
  }
  if (bytes[HAWQ_REGION_CONST] > 0)
    ENG_TRY(cudaMemcpy(e->region[HAWQ_REGION_CONST], plan.constants, (size_t)bytes[HAWQ_REGION_CONST], cudaMemcpyHostToDevice));
  ENG_TRY(cudaMalloc(&e->status_copy, sizeof(int32_t)));
  ENG_TRY(cudaHostAlloc(&e->host_status, sizeof(int32_t), cudaHostAllocDefault));
  *e->host_status = 0;
  for (int k = 0; k < 3; ++k)
    if (plan.present[k])
      if (int rc = capture(e, plan.seq[k], k)) return rc;
  ENG_TRY(cudaDeviceSynchronize());
  return HAWQ_OK;
}

// Runs f with the engine's device current and restores the caller's
template <class Fn>
int on_device(int device, Fn f) {
  int prev = 0;
  ENG_TRY(cudaGetDevice(&prev));
  if (prev != device) ENG_TRY(cudaSetDevice(device));
  const int rc = f();
  if (prev != device) cudaSetDevice(prev);
  return rc;
}

int replay(hawq_engine* e, int k, cudaStream_t s) {
  ENG_TRY(cudaGraphLaunch(e->exec[k], s));
  return HAWQ_OK;
}

}  // namespace

extern "C" {

int hawq_engine_check(const void* data, int64_t bytes, hawq_engine_info* info) {
  Plan plan;
  if (int rc = parse(data, bytes, &plan)) return rc;
  if (info) *info = plan.info;
  return HAWQ_OK;
}

int hawq_engine_load(int device, const void* data, int64_t bytes, hawq_engine** out) {
  if (!out) return fail(HAWQ_ERR_BAD_ARG, "hawq_engine_load: out is null");
  *out = nullptr;
  Plan plan;
  if (int rc = parse(data, bytes, &plan)) return rc;
  hawq_engine* e = new hawq_engine();
  memset(e, 0, sizeof(*e));
  e->device = device;
  e->info = plan.info;
  int prev = 0;
  ENG_TRY(cudaGetDevice(&prev));
  const int rc = load_on(device, plan, e);
  cudaSetDevice(prev);
  if (rc != HAWQ_OK) {
    char msg[512];
    snprintf(msg, sizeof(msg), "%s", hawq_last_error());
    hawq_engine_destroy(e);
    return fail(rc, "%s", msg);
  }
  *out = e;
  return HAWQ_OK;
}

int hawq_engine_destroy(hawq_engine* e) {
  if (!e) return HAWQ_OK;
  on_device(e->device, [&] {
    if (e->stream) cudaStreamSynchronize(e->stream);
    cudaDeviceSynchronize();
    for (int k = 0; k < 3; ++k) {
      if (e->exec[k]) cudaGraphExecDestroy(e->exec[k]);
      if (e->graph[k]) cudaGraphDestroy(e->graph[k]);
    }
    for (int k = 0; k < 4; ++k) cudaFree(e->region[k]);
    cudaFree(e->status_copy);
    cudaFreeHost(e->host_status);
    if (e->stream) cudaStreamDestroy(e->stream);
    hawq_destroy(e->h);
    return HAWQ_OK;
  });
  delete e;
  return HAWQ_OK;
}

void* hawq_engine_input(const hawq_engine* e) { return e ? e->region[HAWQ_REGION_INPUT] : nullptr; }
float* hawq_engine_output(const hawq_engine* e) { return e ? (float*)e->region[HAWQ_REGION_OUTPUT] : nullptr; }

int hawq_engine_get_info(const hawq_engine* e, hawq_engine_info* info) {
  if (!e || !info) return fail(HAWQ_ERR_BAD_ARG, "hawq_engine_get_info: null argument");
  *info = e->info;
  return HAWQ_OK;
}

int hawq_engine_enqueue(hawq_engine* e, void* stream) {
  if (!e) return fail(HAWQ_ERR_BAD_ARG, "hawq_engine_enqueue: null engine");
  return on_device(e->device, [&] { return replay(e, HAWQ_SEQ_FAST, (cudaStream_t)stream); });
}

int hawq_engine_status(const hawq_engine* e, int32_t* flags) {
  if (!e || !flags) return fail(HAWQ_ERR_BAD_ARG, "hawq_engine_status: null argument");
  *flags = *(volatile int32_t*)e->host_status;
  return HAWQ_OK;
}

// CompiledModel._call (hawq_b200/engine.py), rule for rule
int hawq_engine_run(hawq_engine* e, void* stream, int32_t* flags) {
  if (!e) return fail(HAWQ_ERR_BAD_ARG, "hawq_engine_run: null engine");
  const cudaStream_t s = (cudaStream_t)stream;
  return on_device(e->device, [&] {
    if (int rc = replay(e, HAWQ_SEQ_FAST, s)) return rc;
    ENG_TRY(cudaStreamSynchronize(s));
    const int32_t f = *(volatile int32_t*)e->host_status;
    if (flags) *flags = f;
    if (f & HAWQ_FLAG_BAD_RATIO)
      return fail(HAWQ_ERR_RESULT_INVALID, "hawq_engine_run: HAWQ_FLAG_BAD_RATIO raised (a dyadic ratio > 1 reached the fast kernel): results invalid");
    if (f & HAWQ_FLAG_REQUANT_OVERFLOW) {
      ++e->info.fallbacks;
      return replay(e, HAWQ_SEQ_SAFE, s);
    }
    if (e->info.residual_bits == 16 && (f & HAWQ_FLAG_RESIDUAL_OVERFLOW)) {
      ++e->info.fallbacks;
      return replay(e, HAWQ_SEQ_INT32, s);
    }
    return (int)HAWQ_OK;
  });
}

}  // extern "C"
