/* A host without torch: load a denoiser's weights from a raw file, inpaint through include/bdiff.h, write the molecules.
 *
 *   inpaint_main <weights.bin> <tables.bin | -> <mol.bin> <out.bin> <seed> <num_timesteps> <r> <j> <n_0> <n_1> ...
 *
 * weights.bin: as sample_main.c.  tables.bin ("-" = the library's own): float32, bdiff_inpaint's tables_host layout.
 * mol.bin: float32 xh0 [N, 3 + num_h], then uint8 fixed [N].  out.bin: float32 [N, 3 + num_h]. */
#include <stdio.h>
#include <stdlib.h>

#include <cuda_runtime.h>

#include "bdiff.h"

#define CHECK(call)                                                                          \
  do {                                                                                       \
    int rc_ = (call);                                                                        \
    if (rc_ != 0) {                                                                          \
      fprintf(stderr, "%s failed (%d): %s\n", #call, rc_, bdiff_last_error(h));              \
      return 1;                                                                              \
    }                                                                                        \
  } while (0)

static int rd(FILE* f, void* p, size_t n) { return fread(p, 1, n, f) == n; }

int main(int argc, char** argv) {
  bdiff_handle* h = NULL;
  if (argc < 10) { fprintf(stderr, "usage: inpaint_main weights tables mol out seed T r j n...\n"); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  bdiff_config cfg;
  bdiff_sample_config sc = {0};
  int32_t s3[3];
  double d2[2];
  if (!rd(f, &cfg, sizeof cfg) || !rd(f, s3, sizeof s3) || !rd(f, d2, sizeof d2) || !rd(f, sc.norm_values, 12) ||
      !rd(f, sc.norm_biases, 12))
    return 2;
  sc.num_atom_types = s3[0];
  sc.include_charges = s3[1];
  sc.model_timesteps = s3[2];
  sc.schedule_power = d2[0];
  sc.noise_precision = d2[1];
  CHECK(bdiff_create(&cfg, &h));
  int32_t count = 0;
  if (!rd(f, &count, 4)) return 2;
  for (int32_t i = 0; i < count; ++i) {
    int32_t len = 0, ndim = 0;
    char name[256];
    int64_t shape[2] = {1, 1};
    if (!rd(f, &len, 4) || len >= 256 || !rd(f, name, len) || !rd(f, &ndim, 4) || ndim < 1 || ndim > 2 ||
        !rd(f, shape, 8 * ndim))
      return 2;
    name[len] = 0;
    const size_t n = (size_t)shape[0] * (ndim == 2 ? (size_t)shape[1] : 1);
    float* host = (float*)malloc(n * 4);
    float* dev = NULL;
    if (!host || !rd(f, host, n * 4) || cudaMalloc((void**)&dev, n * 4) != cudaSuccess) return 2;
    cudaMemcpy(dev, host, n * 4, cudaMemcpyHostToDevice);
    CHECK(bdiff_set_weight(h, NULL, name, dev, shape, ndim));
    cudaDeviceSynchronize();
    cudaFree(dev);
    free(host);
  }
  fclose(f);
  CHECK(bdiff_weights_missing(h));
  CHECK(bdiff_prepare(h, NULL));
  CHECK(bdiff_sample_setup(h, &sc));

  const unsigned long long seed = strtoull(argv[5], NULL, 10);
  const int T = atoi(argv[6]), r = atoi(argv[7]), j = atoi(argv[8]);
  const int B = argc - 9;
  int32_t* sizes = (int32_t*)malloc(B * 4);
  long long N = 0;
  for (int k = 0; k < B; ++k) N += (sizes[k] = atoi(argv[9 + k]));
  const int ld = 3 + cfg.num_h;
  float* xh0 = (float*)malloc(N * ld * 4);
  uint8_t* fixed = (uint8_t*)malloc(N);
  FILE* m = fopen(argv[3], "rb");
  if (!m || !rd(m, xh0, N * ld * 4) || !rd(m, fixed, N)) return 2;
  fclose(m);
  float* tables = NULL;
  if (argv[2][0] != '-') {      /* the size of the program's tables: a size query of bdiff_repaint_tables */
    int32_t ops = 0, jumps = 0;
    CHECK(bdiff_repaint_tables(&sc, T, r, j, 1, &ops, &jumps, NULL, NULL, NULL, NULL, NULL, NULL, NULL, NULL, NULL, NULL));
    const size_t floats = (size_t)ops * 6 + (size_t)jumps * 4 + 4;
    tables = (float*)malloc(floats * 4);
    FILE* t = fopen(argv[2], "rb");
    if (!t || !rd(t, tables, floats * 4)) return 2;
    fclose(t);
  }
  float* out = NULL;
  if (cudaMalloc((void**)&out, N * ld * 4) != cudaSuccess) return 2;
  CHECK(bdiff_inpaint(h, NULL, B, sizes, NULL, T, r, j, seed, xh0, fixed, 1, tables, out, NULL));
  float* host = (float*)malloc(N * ld * 4);
  cudaMemcpy(host, out, N * ld * 4, cudaMemcpyDeviceToHost);
  FILE* o = fopen(argv[4], "wb");
  if (!o || fwrite(host, 4, N * ld, o) != (size_t)(N * ld)) return 2;
  fclose(o);
  cudaFree(out);
  bdiff_destroy(h);
  free(host);
  free(xh0);
  free(fixed);
  free(sizes);
  free(tables);
  return 0;
}
