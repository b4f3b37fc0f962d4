/* hawq_run: runs a plan file (CompiledModel.save) without Python.
 *
 *   hawq_run PLAN INPUT COUNT OUTPUT [DEVICE]
 *
 * INPUT holds COUNT batches back to back, each exactly the plan's input binding (raw bytes: int8 or uint8 NHWC, or fp32 NCHW);
 * OUTPUT receives COUNT blocks of raw fp32 logits [N, classes].  Every batch goes through hawq_engine_run, the exact forward with the
 * int32 and saturating fallbacks.  Links only libhawq_b200.so and the CUDA runtime. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <cuda_runtime.h>

#include "hawq_b200.h"

static void* read_file(const char* path, long* size) {
  FILE* f = fopen(path, "rb");
  if (!f) return NULL;
  void* buf = NULL;
  if (fseek(f, 0, SEEK_END) == 0 && (*size = ftell(f)) >= 0 && fseek(f, 0, SEEK_SET) == 0) {
    buf = malloc(*size > 0 ? (size_t)*size : 1);
    if (buf && fread(buf, 1, (size_t)*size, f) != (size_t)*size) {
      free(buf);
      buf = NULL;
    }
  }
  fclose(f);
  return buf;
}

static int die(const char* what) {
  fprintf(stderr, "hawq_run: %s\n", what);
  return 1;
}

int main(int argc, char** argv) {
  if (argc < 5 || argc > 6) {
    fprintf(stderr, "usage: %s PLAN INPUT COUNT OUTPUT [DEVICE]\n", argv[0]);
    return 2;
  }
  const long count = strtol(argv[3], NULL, 10);
  const int device = argc == 6 ? atoi(argv[5]) : 0;
  long plan_size = 0, in_size = 0;
  void* plan = read_file(argv[1], &plan_size);
  if (!plan) return die("cannot read the plan file");
  hawq_engine_info info;
  if (hawq_engine_check(plan, plan_size, &info) != HAWQ_OK) return die(hawq_last_error());
  void* input = read_file(argv[2], &in_size);
  if (!input) return die("cannot read the input file");
  if (count < 1 || in_size != count * info.input_bytes) return die("the input file is not COUNT batches of the plan's input binding");
  hawq_engine* eng = NULL;
  if (hawq_engine_load(device, plan, plan_size, &eng) != HAWQ_OK) return die(hawq_last_error());
  free(plan);
  if (cudaSetDevice(device) != cudaSuccess) return die("cudaSetDevice failed");
  const size_t out_bytes = (size_t)(info.output_shape[0] * info.output_shape[1]) * sizeof(float);
  float* logits = (float*)malloc(out_bytes);
  FILE* out = fopen(argv[4], "wb");
  if (!logits || !out) return die("cannot open the output file");
  for (long b = 0; b < count; ++b) {
    if (cudaMemcpy(hawq_engine_input(eng), (const char*)input + b * info.input_bytes, (size_t)info.input_bytes, cudaMemcpyHostToDevice) != cudaSuccess)
      return die("input copy failed");
    int32_t flags = 0;
    if (hawq_engine_run(eng, NULL, &flags) != HAWQ_OK) return die(hawq_last_error());
    if (cudaMemcpy(logits, hawq_engine_output(eng), out_bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return die("output copy failed");
    if (fwrite(logits, 1, out_bytes, out) != out_bytes) return die("cannot write the output file");
  }
  fclose(out);
  hawq_engine_info after;
  hawq_engine_get_info(eng, &after);
  fprintf(stderr, "hawq_run: %ld batches of %lld images, %lld launches per forward, %lld fallbacks\n", count, (long long)info.output_shape[0],
          (long long)info.launches[HAWQ_SEQ_FAST], (long long)after.fallbacks);
  hawq_engine_destroy(eng);
  free(logits);
  free(input);
  return 0;
}
