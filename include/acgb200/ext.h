/*
 * acgb200/ext.h -- entry points that have no counterpart in the reference's
 * headers.  They exist for tests, bench.py and bindings (ctypes cannot size
 * the ABI structs by itself); nothing in the reference driver needs them.
 */
#ifndef ACGB200_EXT_H
#define ACGB200_EXT_H

#include "acgb200/cgcuda.h"

#ifdef __cplusplus
extern "C" {
#endif

/* tunables: "profile" (0/1: CUDA-event timing of each kernel class, fills
 * tgemv/taxpy like the reference's -DACG_ENABLE_PROFILING, acg/cgcuda.c:69-73),
 * "check_every" (iterations between convergence polls), "spmv_lanes",
 * "spmv_nnz_cap", "spmv_rows_cap", "spmv_stages", "spmv_threads", "spmv_unroll",
 * "spmv_max_ctas" (SpMV tile plan overrides, read at acgsolvercuda_init), "spmv_slices"
 * (0/1, default 1: index-free slice-major storage of the rows that repeat a pattern, slices.c; shape
 * overrides "slice_ub", "slice_threads", "slice_max_ctas"), "spmv_symdiag" (1/0, default 1: the slice-covered rows
 * of an exactly symmetric matrix read each stored value once -- the upper diagonals, every lower entry from its
 * mirror row -- when the structure allows, slices.c; "symdiag_evict_first" 0/1 their L2 policy; "symdiag_codes" 1/0,
 * default 1: store them as one-byte codes into a table when they hold at most 256 distinct values), "spmv_merge" (-1/0/1,
 * default -1: merge-path tiles when the row lengths are irregular, mergeplan.c; "merge_items", "merge_threads",
 * "merge_max_ctas"), "pcg_fused" (1/0, default 1: pipelined CG on one GPU runs each iteration's product and
 * vector update in one kernel when the plan has mirrored diagonals and no merge tiles, medium or long rows;
 * "pcg_evict_first" 1/0 the L2 policy of its vector streams; "pcg_group" 2/4/8/16, default 16: it updates p
 * and x once per that many iterations, other values are refused), "spmv_medium", "graph"
 * (0/1: replay groups of iterations as CUDA graphs), "redstream" (0/1: pipelined
 * allreduce on its own stream and communicator; read at acgsolvercuda_init).  Environment variables ACGB200_<KEY> set the
 * same values at first use. */
ACG_API int acgb200_set_option(const char *key, int value);

/* Replace the values of the matrix an initialised solver holds, keeping everything that depends only on the
 * pattern: the tile, slice, mirrored-diagonal and merge plans, row chunks, the halo and peer-memory windows and
 * the multi-vector blocks.  For a sequence of matrices on one pattern (Newton steps, implicit time steps with
 * new coefficients, parameter sweeps), at a fraction of acgsolvercuda_free + acgsolvercuda_init.
 *
 * A is the matrix the solver was built on or another with the same partition and pattern.  Its values are
 * taken as acgsolvercuda_init takes them: from its full storage if it has one (frowptr set), else from the
 * packed triangle, mirrored on the device; either source may be used whichever init used.  After success every
 * product and solve gives what a solver freshly built on A gives under the options in force at the solver's
 * acgsolvercuda_init, with one exception: if A's full storage is not exactly symmetric, a solver holding
 * mirrored diagonals falls back to the slice kernel reading both triangles, as init would, but a later refresh
 * never re-creates mirrored diagonals that init or an earlier refresh dropped.  Whether the diagonals are stored
 * as one-byte codes or as doubles follows the new values, as at init.  Cached CUDA graphs are captured again
 * at the next solve.
 *
 * ACG_ERR_INVALID_VALUE, with the solver left exactly as it was: cg is not a live solver; A has neither full
 * storage nor a packed triangle; the row counts (nrows, nownedrows, ninnerrows, nborderrows, nghostrows,
 * borderrowoffset) or the entry counts differ from init's; or a row pointer or column of either block differs
 * (compared on the device).  ACG_ERR_NOT_SUPPORTED, also before any change: a build without the comparison
 * kernel (host-logic test builds).  A CUDA error after the comparison gives ACG_ERR_CUDA (the third-party code in
 * *errcode, which may be NULL); the solver is then only fit for acgsolvercuda_free.  Local to a rank, with no
 * collective: every rank of a partitioned solver refreshes before its next collective solve. */
ACG_API int acgsolvercuda_update_values(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A, int *errcode);

/* y = A*x through the solver's device matrix: the standalone form of the
 * kernel that replaces cusparseSpMV (acg/cgcuda.c:858).  x, y are HOST arrays
 * of nownedrows doubles (unpartitioned matrices only).  If nrep > 0 the kernel
 * is additionally launched nrep times between two CUDA events on its own
 * stream and the mean duration is returned in milliseconds. */
ACG_API int acgsolvercuda_spmv(struct acgsolvercuda *cg, const double *x, double *y, int nrep, double *ms_per_spmv);

/* One part's share of y = A x on one device with the ghost entries of x supplied by the caller:
 * x has num_nonzeros = owned + ghost entries (host), y the owned rows (host).  path 0: local block +
 * offdiag_kernel on the ghost tail of x (set-up products / NCCL loop, acg/cgcuda.c:858,:878); path 1:
 * the fused tile kernel of the peer-memory loop reading ghosts from a (loop-back) window after the
 * flag wait.  *dot (may be NULL) = sum over owned rows of x_i*y_i from the fused epilogue.  For
 * single-GPU parity tests of the border x ghost path of partitioned matrices. */
ACG_API int acgsolvercuda_spmv_ghost(struct acgsolvercuda *cg, const double *x, double *y, int path, double *dot);

/* The same product in any of the solver's three SpMV epilogue modes (acgsolvercuda_spmv_ghost is
 * mode 1): mode 0 y = A x; mode 1 y = A x and *dot = sum_owned x_i y_i; mode 2 y = b - A x and
 * *dot = sum_owned y_i^2 (b: owned rows, host; may be NULL otherwise).  *dot (may be NULL) is the
 * fused accumulator as the kernels leave it -- 0 in mode 0.  path as above; a whole matrix (no
 * ghosts) takes either.  y is poisoned on the device first, so a row nobody writes comes back NaN.
 * For tests of every SpMV kernel's epilogues against exact products. */
ACG_API int acgsolvercuda_spmv_mode(struct acgsolvercuda *cg, int mode, const double *x, const double *b, double *y,
                                    int path, double *dot);

/* Several right-hand sides of one operator in one pass over the matrix per iteration: nrhs (1..8)
 * independent classic CG recurrences, column j exactly the recurrence acgsolvercuda_solvempi runs for
 * that column alone (its own alpha_j, beta_j, threshold(atol, rtol, ||r0_j||), strict ||r_j|| < tol_j
 * test; a column that meets it stops, its x frozen at that iterate).  Not block CG: the columns share
 * the matrix reads, nothing else.  B and X are host arrays of nownedrows x nrhs doubles, row-major
 * (entry (i, j) at i*nrhs + j); X is the initial guess on entry and the solution on return.  One GPU,
 * unpartitioned matrix: ghost rows or a communicator of more than one rank give ACG_ERR_NOT_SUPPORTED,
 * nrhs outside [1, 8] ACG_ERR_INVALID_VALUE.  Returns ACG_ERR_NOT_CONVERGED if a column with a non-zero
 * tolerance did not converge.  In *cg: niterations is the iterations the loop ran (the maximum over the
 * columns), bnrm2 / r0nrm2 / rnrm2 the Frobenius norms over the columns; stats (may be NULL, nrhs
 * entries) gets each column's own figures. */
struct acgb200_colstats {
    int niterations;            /* iterations this column ran */
    int converged;              /* 1: it met its tolerance (at r0 or later) */
    double bnrm2, r0nrm2, rnrm2;
};
ACG_API int acgsolvercuda_solve_multi(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
                                      int nrhs, const double *B, double *X, int maxits, double residualatol,
                                      double residualrtol, int warmup, struct acgb200_colstats *stats);

/* The multi-vector product of acgsolvercuda_solve_multi in epilogue mode 0 (Y = A X), 1 (Y = A X,
 * dots[j] = x_j.y_j) or 2 (Y = B - A X, dots[j] = y_j.y_j); X, B (mode 2, else may be NULL), Y host
 * arrays of nownedrows x nrhs doubles, row-major; dots (may be NULL) nrhs entries.  Y is poisoned on
 * the device first, so a row no kernel writes comes back NaN.  For tests against exact products. */
ACG_API int acgsolvercuda_spmm_mode(struct acgsolvercuda *cg, int mode, int nrhs, const double *X, const double *B,
                                    double *Y, double *dots);

/* A family of shifted systems (A + shifts[j] I) x_j = b, j < nshifts (1..8), in one Krylov space
 * (multi-shift CG): one classic CG on A -- one single-vector product per iteration for all shifts, no
 * extra dot products -- drives every shifted system through the zeta recurrence, each shift adding
 * two vector updates.  A is the operator the solver holds (with the eps it was built with).  b is a
 * host array of nownedrows doubles; X a host array of nownedrows x nshifts doubles, row-major (entry
 * (i, j) at i*nshifts + j), OUTPUT ONLY: the initial guess is zero for every shift (the method needs
 * collinear initial residuals) and X's contents on entry are ignored.  Shift j stops by the rule
 * acgsolvercuda_solvempi applies to that system alone from x0 = 0: tol = threshold(atol, rtol, ||b||),
 * strict ||r_j|| < tol with ||r_j|| = |zeta_j| ||r|| the recursively updated residual norm; a shift that
 * meets it is frozen at that iterate (0 iterations if ||b|| meets it).  The loop ends when every shift
 * has stopped or at maxits; the seed need not converge itself.  Shifts must be finite and >= 0 (every
 * shifted system then at least as well conditioned as A): anything else, or nshifts outside [1, 8],
 * gives ACG_ERR_INVALID_VALUE.  One GPU, unpartitioned matrix: ghost rows or a communicator of more than
 * one rank give ACG_ERR_NOT_SUPPORTED.  Returns ACG_ERR_NOT_CONVERGED if a shift did not converge under a
 * non-zero tolerance.  In *cg: niterations is the iterations the loop ran, bnrm2 / r0nrm2 / rnrm2 the
 * Frobenius norms over the shifts; stats (may be NULL, nshifts entries) gets each shift's iterations,
 * converged flag, ||b||, r0 = ||b|| and final |zeta_j| ||r||.  `warmup` iterations run first on scratch
 * state; the results do not depend on them. */
ACG_API int acgsolvercuda_solve_shifted(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
                                        int nshifts, const double *shifts, const double *b, double *X,
                                        int maxits, double residualatol, double residualrtol, int warmup,
                                        struct acgb200_colstats *stats);

/* A x = b for symmetric A that may be indefinite or singular: MINRES (Paige & Saunders, SINUM 12, 1975),
 * unpreconditioned, in the formulation of scipy.sparse.linalg.minres.  A is the operator the solver holds
 * (with the eps it was built with); the product is the one the CG solvers use.  b and x are host vectors as
 * in acgsolvercuda_solvempi, x the initial guess on entry and the solution on return.  Stopping rule as
 * acgsolvercuda_solvempi: tol = threshold(atol, rtol, ||r0||), the strict test phi-bar < tol on MINRES's
 * recursively updated residual norm phi-bar, 0 iterations if ||r0|| meets it, ACG_ERR_NOT_CONVERGED by the
 * same rule.  The loop also ends, whatever the tolerance, on an exact Krylov breakdown beta_{k+1} = 0 (after
 * that iteration's update: x is then the minimal-residual solution over an invariant subspace) and on
 * gamma_k = 0, possible only for singular A (before that iteration's update, which is not counted).
 * ||r0|| = 0 runs no iteration; maxits = 0 returns x0 unchanged.  One GPU, unpartitioned matrix: ghost
 * rows or a communicator of more than one rank give ACG_ERR_NOT_SUPPORTED.  In *cg: niterations,
 * bnrm2, r0nrm2, rnrm2 (the final phi-bar), the times and the counters, as for any solve.  `warmup`
 * iterations run first on scratch state; the results do not depend on them. */
ACG_API int acgsolvercuda_solve_minres(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
                                       const struct acgvector *b, struct acgvector *x, int maxits,
                                       double residualatol, double residualrtol, int warmup, int *errcode);

/* A x = b for symmetric positive definite A to an fp64 tolerance with float vectors: CG whose r, p, A p and
 * solution increment y are stored in fp32 (every operation in fp64, each stored value rounded once, scaled
 * by a power of two), with reliable updates (Sleijpen & van der Vorst, Computing 56, 1996; van der Vorst &
 * Ye, SISC 22, 2000): when the fp32 residual has fallen by 0.1 since the last update, or when it meets the
 * tolerance, y is folded into the fp64 x and r is replaced by b - A x from the fp64 product.  Arguments as
 * acgsolvercuda_solve_minres.  tol = threshold(atol, rtol, ||r0||); convergence is only declared on the
 * fp64 residual ||b - A x|| (strict <) of the x returned, and rnrm2 is always that figure, also when the
 * solve stops at maxits (the increment is folded in and the residual recomputed).  ACG_ERR_NOT_CONVERGED
 * follows acgsolvercuda_solvempi's rule.  maxits = 0 returns x0 unchanged; ||r0|| < tol or ||r0|| = 0
 * runs no iteration.  (p, A p) = 0 or non-finite ends the solve before that iteration's update, which is
 * not counted; x is then the last fold.  niterations counts CG steps (fp32 products);
 * acgb200_info.mixed_reliable_updates the reliable updates.  One GPU, unpartitioned matrix: ghost rows or
 * more than one rank give ACG_ERR_NOT_SUPPORTED.  `warmup` iterations run first on scratch state; the
 * results do not depend on them. */
ACG_API int acgsolvercuda_solve_mixed(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
                                      const struct acgvector *b, struct acgvector *x, int maxits,
                                      double residualatol, double residualrtol, int warmup, int *errcode);

/* The fp32 product of acgsolvercuda_solve_mixed on host float vectors over the owned rows: y = fl32(A x),
 * each row's sum formed in fp64 from the widened x, and *dot (may be NULL) = sum x_i y_i in fp64.  y is
 * poisoned on the device first.  One GPU, unpartitioned matrix.  For tests of the fp32 product. */
ACG_API int acgsolvercuda_spmv_f32(struct acgsolvercuda *cg, const float *x, float *y, double *dot);

/* A x = b for symmetric positive definite A by preconditioned CG with M^-1 = p_d(D^-1 A) D^-1 (one GPU).
 *
 * D is the diagonal of the operator the solver holds (the eps of acgsymcsrmatrix_dsymv_init included).
 * z = M^-1 r is formed by d = `degree` steps of Jacobi-scaled Chebyshev iteration on A z = r from z = 0 over
 * the interval [a, b] (Saad, Iterative Methods for Sparse Linear Systems, Alg. 12.1): theta = (a+b)/2,
 * delta = (b-a)/2, sigma = theta/delta, rho_0 = 1/sigma; start res = r, d_0 = D^-1 r / theta, z = d_0; step
 * j = 1..d: res -= A d_{j-1}, rho_j = 1/(2 sigma - rho_{j-1}), d_j = rho_j rho_{j-1} d_{j-1} +
 * (2 rho_j/delta) D^-1 res, z += d_j.  M^-1 is symmetric positive definite exactly when every eigenvalue of
 * D^-1 A lies in (0, a + b), so an underestimated upper bound still gives a valid preconditioner unless it is
 * off by more than a.  degree = 0 is Jacobi PCG (z = D^-1 r); the interval is then ignored and nothing is
 * estimated.  degree outside [0, 16] gives ACG_ERR_INVALID_VALUE.
 *
 * Interval: lmax = 0 estimates b = 1.1 theta_max, theta_max the largest eigenvalue of the Lanczos tridiagonal
 * of 10 Jacobi-PCG steps from r0 on scratch vectors (fewer if the Krylov space breaks down or ||r|| < tol
 * sooner; x and b are not touched).  lmin = 0 sets a = b/10.  A negative or non-finite bound, or a given lmin
 * not below the given or estimated lmax, gives ACG_ERR_INVALID_VALUE before any iteration.
 *
 * Stopping as acgsolvercuda_solvempi: tol = threshold(atol, rtol, ||r0||) and the strict test ||r|| < tol on
 * the recursively updated residual; ||r0|| < tol or ||r0|| = 0 runs no iteration; ACG_ERR_NOT_CONVERGED
 * follows acgsolvercuda_solvempi's rule; maxits = 0 returns x0 unchanged.  (p, A p) <= 0, (r, z) <= 0 or
 * either non-finite ends the solve before that iteration's update, which is not counted.  A diagonal entry
 * that is <= 0 or non-finite gives ACG_ERR_INVALID_VALUE at set-up.  One GPU, unpartitioned matrix: ghost
 * rows or more than one rank give ACG_ERR_NOT_SUPPORTED.  `warmup` iterations run first on scratch state;
 * the results do not depend on them.
 *
 * niterations counts outer iterations (the estimate's steps not included); bnrm2, r0nrm2 and rnrm2 are set
 * as by any solve; the counters count 1 + d products per iteration plus the set-up's and the estimate's.
 * acgb200_info reports the degree, the estimate's steps, a breakdown and the interval used. */
ACG_API int acgsolvercuda_solve_chebyshev(struct acgsolvercuda *cg, const struct acgsymcsrmatrix *A,
                                          const struct acgvector *b, struct acgvector *x, int degree,
                                          double lmin, double lmax, int maxits, double residualatol,
                                          double residualrtol, int warmup, int *errcode);

/* The extreme eigenvalues theta_min <= theta_max of the k x k Lanczos tridiagonal of k CG steps, as
 * acgsolvercuda_solve_chebyshev builds it from its estimate's alpha_j (k of them, > 0) and beta_j (k - 1,
 * >= 0): diagonal 1/alpha_j + beta_{j-1}/alpha_{j-1}, off-diagonal sqrt(beta_j)/alpha_j; Sturm bisection.
 * For tests of the estimate. */
ACG_API int acgb200_cheb_interval_host(int k, const double *alpha, const double *beta, double *theta_min,
                                       double *theta_max);

struct acgb200_info {
    int spmv_lanes_per_row, spmv_rows_cap, spmv_nnz_cap, spmv_stages;
    int spmv_ntiles, spmv_nlong, spmv_grid, spmv_smem_bytes;
    int num_sms;
    int last_launches;          /* kernels + NCCL launches enqueued by the last solve's timed region */
    int last_spmv_count;        /* SpMV applications timed in the last solve (profile=1) */
    double last_spmv_ms;        /* their total device time, CUDA events on the launching stream */
    double last_solve_ms;       /* device time of the last solve window (after the H2D copies and warm-up, to the
                                   end of the loop: the window of tsolve, acg/cgcuda.c:719-722,:1021), CUDA events */
    double last_h2d_ms;         /* host time of the b, x0 upload of the last solve */
    double last_d2h_ms;         /* host time of the x download of the last solve */
    double last_blas_ms;        /* device time of the fused vector-update kernels of the last solve (profile=1) */
    int reserved0;              /* (was: tiles without column indices, a round-1 variant removed after measurement) */
    int64_t spmv_min_bytes;     /* bytes one SpMV launch must move at least, given the plan */
    int spmv_nmedium;           /* rows handled one warp each (option "spmv_medium") */
    int reserved1;              /* (round 1: loop layout, the variants were removed) */
    int spmv_slices;            /* 32-row pattern slices multiplied by spmv_slices_kernel (option "spmv_slices", slices.c) */
    int spmv_slice_rows;        /* rows they cover; the other rows are in tiles */
    int spmv_slice_ub, spmv_slice_grid;
    int spmv_merge_tiles;       /* merge-path tiles (option "spmv_merge", mergeplan.c) ... */
    int spmv_merge_rows;        /* ... the rows [0, spmv_merge_rows) they cover ... */
    int spmv_merge_split;       /* ... and the rows cut by tile boundaries (finished by spmv_merge_fix_kernel) */
    int spmv_slice_exc;         /* rows inside slices that are not in the pattern dictionary (columns from the index array) */
    int spmv_threads, spmv_unroll;              /* shape of the tile kernel (with spmv_lanes_per_row) */
    int spmv_slice_threads;                     /* CTA size of the slice kernel (with spmv_slice_ub) */
    int spmv_merge_threads, spmv_merge_grid, spmv_merge_stages;    /* shape and grid of the merge-path kernel */
    int64_t spmv_slice_value_bytes;             /* slice-major values of the pattern slices, padding included */
    int64_t spmv_slice_nnz;                     /* nonzeros those slices cover (without padding) */
    int spmv_symdiag_diagonals;                 /* upper diagonals stored for the slice-covered rows, whose lower entries
                                                   come from their mirror rows (option "spmv_symdiag"); 0: off */
    int64_t spmv_symdiag_bytes;                 /* their bytes as doubles, zero margins included (with codes the
                                                   device holds spmv_symdiag_code_bytes instead) */
    int pcg_fused;                              /* 1: the last solve was pipelined CG with each iteration's product
                                                   and update fused (option "pcg_fused"); spmv_min_bytes and
                                                   last_spmv_ms then cover the whole iteration, last_blas_ms is 0 */
    int64_t pcg_fused_min_bytes;                /* bytes the fused kernel moves at least: 8 |D| + 96 per slice row
                                                   (|D| + 96 with codes) */
    int spmv_symdiag_codes;                     /* entries of the value table when the stored diagonals are one-byte
                                                   codes into it (option "symdiag_codes"); 0: fp64 diagonals */
    int64_t spmv_symdiag_code_bytes;            /* the codes' bytes, one per element of the diagonals; 0: no codes */
    int mixed_reliable_updates;                 /* reliable updates of the last acgsolvercuda_solve_mixed */
    /* the last acgsolvercuda_solve_chebyshev: its degree, the Jacobi-PCG steps of the interval estimate (0: none
     * ran), 1 if a breakdown ended it, and the interval [cheb_lmin, cheb_lmax] used (0, 0: none) */
    int cheb_degree, cheb_est_iterations, cheb_breakdown;
    double cheb_lmin, cheb_lmax;
    int pcg_group;                              /* the group of the last solve if it was fused pipelined CG (option
                                                   "pcg_group"), 0 otherwise */
};
ACG_API int acgsolvercuda_info(const struct acgsolvercuda *cg, struct acgb200_info *info);

/* The SpMV tile plan acgsolvercuda_init would build for a CSR row-pointer array
 * (int64, nrows+1 entries), computed on the host without a device: tiles4 gets
 * {row_begin, nrows, k_al, nnz_al} per tile, longrows the rows that exceed a
 * tile; info->spmv_* describe the plan.  For tests of the host logic. */
ACG_API int acgb200_spmv_plan_host(int nrows, const int64_t *rowptr, struct acgb200_info *info,
                                   int *tiles4, int maxtiles, int *longrows, int maxlong);
/* same, and with colidx != NULL (0-based) also the pattern slices: the tiles then skip the rows of
 * covered slices; info->spmv_slices / spmv_slice_rows count them (acgb200_slices_host lists them) */
ACG_API int acgb200_spmv_plan_host2(int nrows, const int64_t *rowptr, const int *colidx, struct acgb200_info *info,
                                    int *tiles4, int maxtiles, int *longrows, int maxlong);

/* The pattern-slice plan of a 0-based CSR matrix (slices.c), host only: slices4 gets {row0, nrows,
 * len, vblk} per covered slice (at most maxslices), covered one byte per 32-row slice, totals
 * {nslices, value blocks of 32 doubles, nonzeros covered, rows covered, row stride of the padded
 * offset table, patterns in the table}, spatoff (8192 ints) the zero-padded offset table, patid (nrows, may be
 * NULL) the pattern id per row as the slice kernel sees it (0xFFFF: exception row, columns from the index array),
 * exc2 (may be NULL) {exception rows inside slices, their nonzeros}.  Rows [0,cover_hi) are eligible. */
ACG_API int acgb200_slices_host(int nrows, int cover_hi, const int64_t *rowptr, const int *colidx,
                                int *slices4, int maxslices, unsigned char *covered, int64_t *totals6, int *spatoff,
                                unsigned short *patid, int64_t *exc2);

/* The mirrored-diagonal plan of the pattern slices of a 0-based CSR matrix (slices.c), host only: info5 gets
 * {reason (0: eligible; 1 no slices, 2 exception rows, 3 a covered row not sorted, 4 more than 64 offsets,
 * 5 no fewer bytes, 6 too large), |O|, |D|, zero margin, stride}, o the offsets O of the covered rows (64 ints),
 * d the stored diagonals D (64 ints), tab2 {value offset, column offset} per entry of O (128 ints; eligible
 * plans only): entry e of covered row i is value tab2[2e] + i of the diagonals -- diagonal D[k] at
 * [k * stride, (k+1) * stride), a[j, j + D[k]] at margin + j -- times x[i + tab2[2e+1]].  acgsolvercuda_init
 * uses the layout if this says eligible and the values pass a bitwise symmetry check on the device.  Rows
 * [0,cover_hi) are eligible for slices. */
ACG_API int acgb200_symdiag_host(int nrows, int cover_hi, const int64_t *rowptr, const int *colidx, int *info5,
                                 int *o, int *d, int *tab2);

/* acgsymcsrmatrix_dsymv_init (acg/symcsrmatrix.c:760-851) computed on the current CUDA device
 * (expand.cu): the packed triangle is uploaded, mirrored there into the full local block and the
 * border x ghost block, and copied back into A -- arrays byte-identical to the host routine's.
 * ACG_ERR_CUDA without a device (the host routine is the one to call then).  Programs that only
 * want to solve need not call either: acgsolvercuda_init expands on the device by itself when the
 * matrix has no full storage (diagonal shift 0), which also halves the matrix upload. */
ACG_API int acgsymcsrmatrix_dsymv_init_cuda(struct acgsymcsrmatrix *A, double eps, int *cudaerrcode);

/* The merge-path tile plan of rows [0,hi) of a CSR row-pointer array (mergeplan.c), host only: tiles4 gets
 * {r0, nre, k0, nnz} per tile (at most maxtiles), split3 {row, ta, tb} per row cut by tile boundaries (at
 * most maxtiles); *ntiles, *nsplit the counts. */
ACG_API int acgb200_merge_plan_host(int hi, const int64_t *rowptr, int items, int *tiles4, int maxtiles,
                                    int *split3, int *ntiles, int *nsplit);

/* One part of the block-partitioned 7- or 27-point stencil matrix on an
 * nx*ny*nz box (diag 6 / 26, neighbours -1, lexicographic numbering, px*py*pz
 * geometric blocks, part = bi + px*(bj + py*bk)), built directly without a
 * global matrix: array-for-array what acgsymcsrmatrix_partition yields for that
 * part (stencil.c).  Follow with acgsymcsrmatrix_dsymv_init. */
ACG_API int acgb200_stencil_part(int kind, int nx, int ny, int nz, int px, int py, int pz, int part,
                                 struct acgsymcsrmatrix *A);

/* R-MAT style power-law SPD matrix (BASELINE config 5): n vertices, `nedges`
 * draws with quadrant probabilities abcd (NULL: 0.57, 0.19, 0.19, 0.05),
 * symmetrised, deduplicated, off-diagonal -1, diagonal degree+1.  Threaded; the
 * result does not depend on the thread count (rmat.c). */
ACG_API int acgb200_rmat_spd(int64_t n, int64_t nedges, uint64_t seed, const double *abcd,
                             struct acgsymcsrmatrix *A);

/* Geometric row -> part map of an nx*ny*nz lexicographic grid in px*py*pz blocks
 * (the partition acgb200_stencil_part assumes; the alternative to the METIS call
 * of acg/graph.c:510 when the geometry is known), and the most cubic
 * factorisation px <= py <= pz of a part count. */
ACG_API int acgb200_partition_rows_grid(int nx, int ny, int nz, int px, int py, int pz, int *rowparts);
ACG_API void acgb200_grid_factors(int nparts, int *px, int *py, int *pz);

/* Matrix Market ingest (mtxfile.c): text, and aCG's binary encoding -- header and
 * size line as text, then rowidx[nnz], colidx[nnz] (1-based acgidx_t), a[nnz]
 * (double); acg/mtxfile.c:1107-1127, written by mtx2bin (mtx2bin/mtx2bin.c:538-549),
 * read by `acg-cuda --binary` (cuda/acg-cuda.c:1297-1304).  Only "matrix
 * coordinate real symmetric" files are accepted.  Matrices come out 0-based. */
struct acgb200_mtxinfo {
    int64_t nrows, ncols, nnzs;
    int64_t data_offset;      /* first byte after the size line */
    int field;                /* 0 real, 1 integer, 2 pattern, 3 other */
    int symmetric;
};
ACG_API int acgb200_mtx_info(const char *path, struct acgb200_mtxinfo *info);
ACG_API int acgb200_mtx_read(const char *path, int binary, struct acgsymcsrmatrix *A);
/* Part `part` of the row partition `rowparts` (nrows entries in [0,nparts)) of a
 * binary file, array for array what acgsymcsrmatrix_partition returns for that
 * part, without any process holding the whole matrix: the file is streamed and
 * only entries with an end in `part` are kept -- the per-rank replacement of the
 * reference's read-on-root + scatter (cuda/acg-cuda.c:1516-1782). */
ACG_API int acgb200_mtx_read_part(const char *path, int nparts, const int *rowparts, int part,
                                  struct acgsymcsrmatrix *A);

/* Row p of the communication matrix (cuda/acg-cuda.c:1713-1775, the driver's
 * --output-comm-matrix): row[q] = border values part A sends to part q per halo
 * exchange; nparts entries. */
ACG_API int acgb200_comm_matrix_row(const struct acgsymcsrmatrix *A, int nparts, int64_t *row);

/* Row-pattern dictionary of a 0-based CSR matrix (host logic of the pattern
 * slices, compress.c).  patptr needs max_entries+1 ints (at most that many
 * patterns), patoff max_entries ints, patid nrows entries; 0xFFFF in patid
 * marks a row whose pattern is not in the dictionary. */
ACG_API int acgb200_patterns_host(int nrows, const int64_t *rowptr, const int *colidx, int max_entries,
                                  int *npat, int *nentries, int *patptr, int *patoff, unsigned short *patid,
                                  int64_t *nmatched);

/* Inverse send map of the peer-memory halo exchange (host logic of p2p.c): for
 * border row b, entries [bptr[b], bptr[b+1]) give the recipient index bq[e] and
 * the destination offset bdst[e] in that recipient's ghost buffer;
 * rdispl_at_recipient[i] is recipient i's receive displacement for this sender.
 * bptr: nborder+1 ints, bq/bdst: halo->sendsize ints. */
ACG_API int acgb200_p2p_inverse_map(const struct acghalo *halo, int borderoff, int nborder,
                                    const int *rdispl_at_recipient, int *bptr, int *bq, int *bdst);

/* struct sizes, for bindings: "acgsolvercuda", "acgsymcsrmatrix", "acgvector",
 * "acgcomm", "acghalo"; returns 0 for unknown names */
ACG_API size_t acgb200_sizeof(const char *name);
/* 1 if this build was compiled with ACG_HAVE_MPI (struct acgcomm then has the
 * MPI member), else 0 */
ACG_API int acgb200_have_mpi(void);

/* page-lock / unlock caller-owned host memory (b->x, x->x) so that the solver's
 * H2D/D2H copies run at full PCIe speed; optional, the solve works on pageable memory */
ACG_API int acgb200_host_register(void *ptr, size_t bytes);
ACG_API int acgb200_host_unregister(void *ptr);

/* NCCL bootstrap for hosts without MPI (the reference driver broadcasts the
 * unique id over MPI, cuda/acg-cuda.c:1104-1122; bench.py / tests broadcast
 * these 128 bytes over torch.distributed instead) */
ACG_API int acgb200_nccl_unique_id(void *id128);
ACG_API int acgb200_comm_init_rank(struct acgcomm *comm, int nranks, const void *id128, int rank, int *ncclerrcode);
ACG_API int acgb200_comm_destroy(struct acgcomm *comm);

#ifdef __cplusplus
}
#endif
#endif
