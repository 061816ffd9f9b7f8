/*
 * plan.c -- host-only parts of the SpMV tile plan: the heuristic that picks the
 * tile shape and the byte count a launch must move at least.  No CUDA calls
 * (the occupancy-dependent grid size is set by acgb200_spmv_configure in
 * kernels.cu).
 */
#include "internal.h"

#define SPMV_THREADS 128

/* bytes per stored element of the mirrored diagonals: a double, or a one-byte code */
static int64_t symdiag_elem_bytes(const struct acgb200_spmvplan *pl) { return pl->symdiag_codes > 0 ? 1 : 8; }

int64_t acgb200_spmv_min_bytes(const struct acgb200_spmvplan *pl)
{
    /* tiles: values + indices + per row: row pointer, y, x; slices: padded values + per row: pattern id, y, x */
    const int64_t tnnz = pl->nnz - pl->slice_nnz, trows = pl->nrows - pl->slice_rows;
    /* mirrored diagonals: per covered row one value (8 bytes, or a 1-byte code) per stored diagonal (the lower
     * entries come again from L2), y, x */
    if (pl->symdiag_nd > 0)
        return tnnz * 12 + trows * 20 + (int64_t) pl->slice_rows * (symdiag_elem_bytes(pl) * pl->symdiag_nd + 16);
    return tnnz * 12 + trows * 20 + pl->sval_blocks * 256 + (int64_t) pl->slice_rows * 18
           + pl->slice_excnnz * 4 + pl->slice_exc * 8;
}

/* fused pipelined CG with every update done in its own iteration, per covered row: the stored diagonals,
 * w_i, reads of z t p r x, writes of z t p x r w' */
int64_t acgb200_pcg_fused_min_bytes(const struct acgb200_spmvplan *pl)
{
    return (int64_t) pl->slice_rows * (symdiag_elem_bytes(pl) * pl->symdiag_nd + 96);
}

/* the whole fused iteration as it runs, p and x updated once per group of m iterations: the tile kernel's
 * product, then per row the mean over a group.  Covered rows: w_i, z t r read, z t r w' written (64) in
 * every iteration, and in the group's last one a pass that reads the group's m r's and p x and writes p x,
 * so 64 + (32 + 8 m) / m = (72 m + 32) / m on average.  Tile rows: q_i read on top. */
int64_t acgb200_pcg_iteration_min_bytes(const struct acgb200_spmvplan *pl, int m)
{
    const int64_t tnnz = pl->nnz - pl->slice_nnz, trows = pl->nrows - pl->slice_rows;
    return tnnz * 12 + trows * 20 + (trows * (80 * (int64_t) m + 32)) / m
           + (int64_t) pl->slice_rows * symdiag_elem_bytes(pl) * pl->symdiag_nd
           + ((int64_t) pl->slice_rows * (72 * (int64_t) m + 32)) / m;
}

/*
 * Tile-plan heuristic, from sweeps of tile shapes (tools/sweep.py).  The
 * compute phase of a tile is a chain LDS(col) -> LDG(x) -> DFMA per nonzero and
 * ptxas keeps only ~2 gathers in flight per thread, so throughput comes from
 * resident warps: small stages (0.5-1k nonzeros, 6-11 KiB) let 10-18 CTAs of 128
 * threads share an SM.  Deeper TMA rings lower the CTA count and lose.
 *   lanes per row G : largest power of two with mean row length / G >= 4
 *   rows per tile   : T / G   (one pass per tile)
 *   nonzeros/tile   : rows * longest row for near-uniform rows (stencils),
 *                     else twice the mean -- rows longer than that take the
 *                     long-row path
 */
void acgb200_spmv_choose(struct acgb200_spmvplan *pl, int nrows, int64_t nnz, int64_t maxrowlen)
{
    const double avg = nrows > 0 ? (double) nnz / nrows : 0.0;
    int G = 1;
    while (G < 32 && avg / (2 * G) >= 4.0) G *= 2;
    const int T = SPMV_THREADS;
    const int rows_cap = T / G;
    int64_t cap = (int64_t) (2.0 * avg * rows_cap) + 8;
    if (maxrowlen > 0 && (double) maxrowlen <= 2.0 * avg + 8.0) cap = maxrowlen * rows_cap;
    if (cap < 256) cap = 256;
    if (cap > 6144) cap = 6144;
    pl->nrows = nrows; pl->nnz = nnz;
    pl->lanes_per_row = G; pl->rows_cap = rows_cap; pl->nnz_cap = (int) ((cap + 3) & ~(int64_t) 3);
    pl->nstages = 2; pl->threads = T; pl->unroll = 8;
    pl->long_chunks = 8;
}

