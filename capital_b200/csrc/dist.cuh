// Multi-GPU side of the path: the distributed schedules over the peer layer (peer.cuh), one process per GPU.
#pragma once
#include "common.cuh"

void dist_destroy(capital_ctx* ctx);
capital_status_t dist_release_peer_maps(capital_ctx* ctx);  // collective: unmap / free the peer arena (capital_release_workspace)
capital_status_t dist_cholinv_factor(capital_ctx* ctx, const double* A_local, int64_t n, const capital_cholinv_args_t* args,
                                     capital_structure_t ostruct, double* R_local, double* Rinv_local);
capital_status_t dist_cholinv_residual(capital_ctx* ctx, const double* A_local, int64_t n, capital_structure_t structure,
                                       const double* R_local, double* residual);
// what the solve computes: A^-1 B (both halves), or one half alone: R^-1 B or R^-T B (capital_cholinv_apply_rinv_f64), or a product
// with the factor itself: R B or R^T B (capital_cholinv_apply_r_f64)
enum { SOLVE_FULL = 0, SOLVE_RINV = 1, SOLVE_RINVT = 2, SOLVE_R = 3, SOLVE_RT = 4 };
capital_status_t dist_cholinv_solve(capital_ctx* ctx, int64_t n, const capital_cholinv_args_t* args, capital_structure_t structure,
                                    const double* R_local, const double* Rinv_local, int64_t nrhs, const double* B, int64_t ldb,
                                    double* X, int64_t ldx, int mode);
capital_status_t dist_cholinv_inverse(capital_ctx* ctx, int64_t n, const capital_cholinv_args_t* args, capital_structure_t structure,
                                      const double* R_local, const double* Rinv_local, double* Ainv_local);
capital_status_t dist_cholinv_sygst(capital_ctx* ctx, int64_t n, const capital_cholinv_args_t* args, capital_structure_t structure,
                                    const double* R_local, const double* Rinv_local, const double* A_local, double* C_local);
capital_status_t dist_cholinv_sygst_ab(capital_ctx* ctx, int64_t n, const capital_cholinv_args_t* args, capital_structure_t structure,
                                       const double* R_local, const double* A_local, double* C_local);
capital_status_t dist_cholinv_inverse_residual(capital_ctx* ctx, const double* A_local, int64_t n, capital_structure_t structure,
                                               const double* Ainv_local, double* residual);
capital_status_t dist_cacqr_factor(capital_ctx* ctx, const double* A_local, int64_t m, int64_t n, int num_iter,
                                   const capital_cholinv_args_t* ci_args, capital_structure_t rstruct, double* Q_local, double* R_local);
capital_status_t dist_cacqr_apply_qt(capital_ctx* ctx, int64_t m, int64_t n, const double* Q_local, capital_structure_t rstruct,
                                     const double* R_local, int64_t nrhs, const double* B_local, int64_t ldb, double* X, int64_t ldx);
capital_status_t dist_cacqr_apply_q(capital_ctx* ctx, int64_t m, int64_t n, const double* Q_local, int64_t nrhs, const double* Z,
                                    int64_t ldz, double* C_local, int64_t ldc);
capital_status_t dist_cacqr_residual(capital_ctx* ctx, const double* A_local, int64_t m, int64_t n, const double* Q_local,
                                     capital_structure_t rstruct, const double* R_local, double* residual, double* orthogonality);

// batched CholeskyQR on this context's GPU (arguments checked by the C entry points)
capital_status_t dist_cacqr_factor_batched(capital_ctx* ctx, int64_t m, int64_t n, int64_t batch, int num_iter, const double* A, double* Q,
                                           double* R, int* info);
capital_status_t dist_cacqr_lstsq_batched(capital_ctx* ctx, int64_t m, int64_t n, int64_t batch, const double* Q, const double* R,
                                          int64_t nrhs, const double* B, double* X);

capital_status_t dist_summa_gemm_tn(capital_ctx* ctx, int64_t m, int64_t n, int64_t k, double alpha, const double* A_local,
                                    const double* B_local, double beta, double* C_local);

// helpers shared with api.cu
bool cap_is_device_ptr(const void* p);
capital_status_t cap_stage_in(capital_ctx* ctx, const double* src, size_t count, const char* name, const double** out);
capital_status_t cap_stage_out_begin(capital_ctx* ctx, double* dst, size_t count, const char* name, double** dev);
capital_status_t cap_stage_out_end(capital_ctx* ctx, double* dst, size_t count, const double* dev);
capital_status_t cap_check_info(capital_ctx* ctx);
