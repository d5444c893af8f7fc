/* Plain C caller of the C ABI -- the same positional arguments and protocol as the reference's bench/cholesky/cholinv.cpp
 * (:14-22 argv, :38-60 warm-up + timed factor + "total time" line), single process / single GPU, HOST buffers (the library
 * stages H2D / D2H itself, so this file needs no CUDA header):
 *
 *     gcc -O2 -Iinclude examples/cholinv_driver.c -Lcapital_b200 -lcapital_b200 -Wl,-rpath,$PWD/capital_b200 -lm -o cholinv_driver
 *     ./cholinv_driver num_rows rep_div complete_inv split bcMultiplier layout num_chunks num_iter
 */
#include <stdio.h>
#include <stdlib.h>
#include <time.h>
#include "capital_b200.h"

static double now(void) { struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec + 1e-9 * t.tv_nsec; }

int main(int argc, char** argv) {
  if (argc < 9) { fprintf(stderr, "usage: %s num_rows rep_div complete_inv split bcMultiplier layout num_chunks num_iter\n", argv[0]); return 2; }
  const int64_t n = atoll(argv[1]);
  capital_cholinv_args_t args = {atoll(argv[3]), atoll(argv[4]), atoll(argv[5]), 'U'};
  const int layout = atoi(argv[6]), num_chunks = atoi(argv[7]), num_iter = atoi(argv[8]);
  capital_grid_t grid;
  if (capital_grid_square(1, 0, 1, layout, num_chunks, &grid) != CAPITAL_OK) { fprintf(stderr, "bad grid\n"); return 1; }
  capital_ctx* ctx = NULL;
  if (capital_create(&ctx, &grid, 0, NULL) != CAPITAL_OK) { fprintf(stderr, "capital_create failed: no sm_90 device (there is no CPU fallback)\n"); return 1; }
  const size_t tri = (size_t)n * (n + 1) / 2;
  double* A = (double*)malloc(sizeof(double) * n * n);
  double* R = (double*)malloc(sizeof(double) * tri);
  double* Rinv = (double*)malloc(sizeof(double) * tri);
  if (!A || !R || !Rinv) return 1;
  if (capital_distribute_symmetric_f64(ctx, A, n, 1) != CAPITAL_OK) { fprintf(stderr, "%s\n", capital_last_error(ctx)); return 1; }
  if (capital_cholinv_factor_f64(ctx, A, n, &args, CAPITAL_UPPERTRI_PACKED, R, Rinv) != CAPITAL_OK) {  /* warm-up, :44 */
    fprintf(stderr, "%s\n", capital_last_error(ctx)); return 1;
  }
  for (int i = 0; i < num_iter; i++) {
    const double t0 = now();
    if (capital_cholinv_factor_f64(ctx, A, n, &args, CAPITAL_UPPERTRI_PACKED, R, Rinv) != CAPITAL_OK) { fprintf(stderr, "%s\n", capital_last_error(ctx)); return 1; }
    printf("total time - %g\n", now() - t0);  /* :59 */
  }
  double res = -1.0;
  if (capital_cholinv_residual_f64(ctx, A, n, CAPITAL_UPPERTRI_PACKED, R, &res) != CAPITAL_OK) { fprintf(stderr, "%s\n", capital_last_error(ctx)); return 1; }
  printf("%g\n", res);  /* the residual block the reference keeps commented out, :61-66 */
  capital_destroy(ctx);
  free(A); free(R); free(Rinv);
  return res < 1e-12 ? 0 : 3;
}
