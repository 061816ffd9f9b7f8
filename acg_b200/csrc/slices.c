/*
 * slices.c -- host plan of the "pattern slices" of the SpMV (no CUDA calls).
 *
 * Matrices from stencils repeat a few row patterns (compress.c: the sequence of
 * offsets col - row; 27 patterns describe the 27-point stencil on a box).  For
 * 32 consecutive rows that are all in the dictionary neither column indices nor
 * row pointers are needed: a 2-byte pattern id per row gives the row's length and
 * its columns.  Such a slice is stored slice-major -- entry slot e of the 32 rows
 * in 32 consecutive doubles, rows shorter than the slice's longest padded with
 * zeros -- so that a warp with one row per lane reads the matrix with perfectly
 * coalesced 256-byte loads straight from HBM, 8 bytes per nonzero, and needs no
 * shared-memory staging at all (spmv_slices_kernel).  A row's products are added
 * in the row's CSR order, one accumulator.
 *
 * A slice may hold a few rows that are NOT in the dictionary ("exception rows", at
 * most SLICE_MAXEXC of its 32): inside a partition's block every grid line has one
 * row next to the border shell whose offsets to the separately numbered border rows
 * are unique to it -- 1.5 % of the interior rows at 8 parts, but one in 29 % of all
 * aligned 32-row runs.  Their values are slice-major like everybody's; only their
 * columns come from the CSR index array (spmv_slices_kernel<.., EXC>), so such a
 * slice still streams 8 bytes per nonzero instead of falling back to tiles.
 *
 * Rows outside covered slices (runs with many unmatched rows, the border rows between
 * GPUs, the ragged end) stay with the TMA tile kernel; the tile planner skips covered
 * slices (cut_tiles in cgcuda.c).  An unstructured matrix ends up with no slices and
 * pays nothing.
 */
#include "acgb200/error.h"
#include "internal.h"

#include <stdlib.h>
#include <string.h>

#define SLICE_ROWS 32
#define SLICE_MAXLEN 64          /* longest row a slice may hold */
#define SLICE_TABLE_MAX 8192     /* ints in the padded offset table (32 KiB of shared memory) */
#define SLICE_MAXEXC 8           /* rows of a slice that may take their columns from the index array */

void acgb200_sliceplan_free(struct acgb200_sliceplan *sp)
{
    free(sp->slices); free(sp->covered); free(sp->spatoff); free(sp->patid);
    memset(sp, 0, sizeof(*sp));
}

int acgb200_slices_plan(int nrows, int cover_hi, const int64_t *rowptr, const struct acgb200_patterns *pat,
                        struct acgb200_sliceplan *out)
{
    memset(out, 0, sizeof(*out));
    const int nsl_all = (nrows + SLICE_ROWS - 1) / SLICE_ROWS;
    out->covered = calloc((size_t) (nsl_all > 0 ? nsl_all : 1), 1);
    if (!out->covered) return ACG_ERR_ERRNO;
    if (!pat || pat->npat <= 0 || cover_hi < SLICE_ROWS) return ACG_SUCCESS;
    if (cover_hi > nrows) cover_hi = nrows;
    const int nfull = cover_hi / SLICE_ROWS;
    /* longest pattern that may enter a slice, and the table it implies */
    int lpad = 0;
    for (int p = 0; p < pat->npat; p++) {
        const int len = pat->patptr[p + 1] - pat->patptr[p];
        if (len <= SLICE_MAXLEN && len > lpad) lpad = len;
    }
    if (lpad <= 0) return ACG_SUCCESS;
    /* the table holds the most frequent patterns that fit (ids are by descending frequency); rows with other
     * patterns count as exception rows */
    const int idmax = (int64_t) pat->npat * lpad > SLICE_TABLE_MAX ? SLICE_TABLE_MAX / lpad : pat->npat;
    out->patid = malloc((size_t) (nrows > 0 ? nrows : 1) * sizeof(*out->patid));
    if (!out->patid) { acgb200_sliceplan_free(out); return ACG_ERR_ERRNO; }
    for (int r = 0; r < nrows; r++) {
        const unsigned short id = pat->patid[r];
        out->patid[r] = (id != ACGB200_NOPATTERN && id < idmax && pat->patptr[id + 1] - pat->patptr[id] <= lpad)
                            ? id : (unsigned short) ACGB200_NOPATTERN;
    }
    out->slices = malloc((size_t) (nfull > 0 ? nfull : 1) * sizeof(*out->slices));
    if (!out->slices) { acgb200_sliceplan_free(out); return ACG_ERR_ERRNO; }
    int64_t lenhist[SLICE_MAXLEN + 1];
    memset(lenhist, 0, sizeof(lenhist));
    int ns = 0;
    int64_t blocks = 0, nnz = 0, nexc = 0, excnnz = 0;
    for (int s = 0; s < nfull; s++) {
        const int r0 = s * SLICE_ROWS;
        int ok = 1, L = 0, exc = 0;
        int64_t cnt = 0, ecnt = 0;
        for (int r = r0; r < r0 + SLICE_ROWS && ok; r++) {
            const int64_t len = rowptr[r + 1] - rowptr[r];
            if (len > SLICE_MAXLEN) { ok = 0; break; }
            if (out->patid[r] == ACGB200_NOPATTERN) { if (++exc > SLICE_MAXEXC) { ok = 0; break; } ecnt += len; }
            if (len > L) L = (int) len;
            cnt += len;
        }
        /* padding may not cost more than the column indices saved (12 -> 8 bytes per nonzero) */
        if (!ok || L == 0 || 8 * (int64_t) SLICE_ROWS * L > 11 * cnt) continue;
        if (blocks + L > INT32_MAX) break;
        out->covered[s] = 1;
        out->slices[ns].row0 = r0; out->slices[ns].nrows = SLICE_ROWS; out->slices[ns].len = L;
        out->slices[ns].vblk = (int) blocks;
        blocks += L; nnz += cnt; ns++; nexc += exc; excnnz += ecnt;
        for (int r = r0; r < r0 + SLICE_ROWS; r++) lenhist[rowptr[r + 1] - rowptr[r]]++;
    }
    /* worth a second kernel only if it takes most of the rows */
    if ((int64_t) ns * SLICE_ROWS * 2 < cover_hi) {
        memset(out->covered, 0, (size_t) nsl_all);
        free(out->slices); out->slices = NULL;
        free(out->patid); out->patid = NULL;
        return ACG_SUCCESS;
    }
    out->nslices = ns; out->blocks = blocks; out->nnz = nnz; out->rows = ns * SLICE_ROWS;
    out->lpad = lpad; out->npat = idmax; out->nexc = nexc; out->excnnz = excnnz;
    int dom = 1;
    for (int l = 1; l <= SLICE_MAXLEN; l++) if (lenhist[l] > lenhist[dom]) dom = l;
    out->domlen = dom;
    out->spatoff = calloc((size_t) idmax * (size_t) lpad, sizeof(int));
    if (!out->spatoff) { acgb200_sliceplan_free(out); return ACG_ERR_ERRNO; }
    for (int p = 0; p < idmax; p++) {
        const int len = pat->patptr[p + 1] - pat->patptr[p];
        if (len > lpad) continue;                       /* never referenced by a covered row */
        memcpy(out->spatoff + (size_t) p * lpad, pat->patoff + pat->patptr[p], (size_t) len * sizeof(int));
    }
    return ACG_SUCCESS;
}

/*
 * Mirrored diagonals.  The matrix is symmetric and its full storage mirrors the packed triangle, so
 * a[i, i+o] with o < 0 is a bit-for-bit copy of a[i+o, i], the entry at offset -o of row i+o.  Of the
 * covered rows' offsets O only D = {|o|} need storing: diagonal d holds a[j, j+d] of every owned row j
 * (0 where row j has no such entry), behind a zero margin of at least max D entries.  A covered row then
 * reads entry o from diagonal |o| at row i (o >= 0) or at its mirror row i+o (o < 0), for o in O
 * ascending -- its CSR order, with zeros where it has no entry (spmv_symdiag_kernel).  Rows with the same
 * pattern id have the same offsets, so the patterns the covered rows use give O.
 */
_Static_assert(ACGB200_SYMDIAG_MAX == SLICE_MAXLEN, "mirrored diagonals hold the rows a slice may hold");

int acgb200_symdiag_plan(int nrows, const struct acgb200_sliceplan *sp, const struct acgb200_patterns *pat,
                         struct acgb200_symdiag *out)
{
    memset(out, 0, sizeof(*out));
    if (!sp || sp->nslices <= 0 || !pat || !sp->patid) { out->reason = SYMDIAG_NO_SLICES; return ACG_SUCCESS; }
    if (sp->nexc > 0) { out->reason = SYMDIAG_EXCEPTIONS; return ACG_SUCCESS; }
    unsigned char *used = calloc((size_t) sp->npat + 1, 1);
    if (!used) return ACG_ERR_ERRNO;
    for (int s = 0; s < sp->nslices; s++)
        for (int r = sp->slices[s].row0; r < sp->slices[s].row0 + sp->slices[s].nrows; r++) used[sp->patid[r]] = 1;
    int no = 0;
    for (int p = 0; p < sp->npat && !out->reason; p++) {
        if (!used[p]) continue;
        const int *off = pat->patoff + pat->patptr[p];
        const int len = pat->patptr[p + 1] - pat->patptr[p];
        for (int k = 0; k < len && !out->reason; k++) {
            if (k > 0 && off[k] <= off[k - 1]) { out->reason = SYMDIAG_UNSORTED; break; }
            int lo = 0;                                 /* insert off[k] into the sorted O */
            while (lo < no && out->o[lo] < off[k]) lo++;
            if (lo < no && out->o[lo] == off[k]) continue;
            if (no == ACGB200_SYMDIAG_MAX) { out->reason = SYMDIAG_TOO_MANY; break; }
            memmove(out->o + lo + 1, out->o + lo, (size_t) (no - lo) * sizeof(int));
            out->o[lo] = off[k]; no++;
        }
    }
    free(used);
    if (out->reason) return ACG_SUCCESS;
    out->no = no;
    /* D: the absolute values, ascending (O is sorted, so merge its negative part reversed with the rest) */
    int nd = 0, neg = 0;
    while (neg < no && out->o[neg] < 0) neg++;
    for (int a = neg - 1, b = neg; a >= 0 || b < no;) {
        const int v = (b >= no || (a >= 0 && -out->o[a] <= out->o[b])) ? -out->o[a--] : out->o[b++];
        if (nd == 0 || out->d[nd - 1] != v) out->d[nd++] = v;
    }
    out->nd = nd;
    /* the stored diagonals replace the slice-major values: 8|D| bytes per covered row against 256 per block */
    if ((int64_t) nd * sp->rows >= sp->blocks * 32) { out->reason = SYMDIAG_NO_GAIN; return ACG_SUCCESS; }
    /* 32-bit value offsets in the kernel */
    if ((int64_t) nd * ((int64_t) nrows + out->d[nd - 1] + 64) > INT32_MAX) out->reason = SYMDIAG_TOO_LARGE;
    return ACG_SUCCESS;
}

/* Where the kernel finds entry e of a covered row i: diagonal d sits at [idx(d) * stride, + stride) with
 * a[j, j+d] at margin + j; entry o is value voff + i and column i + coff (coff = o).  The margin and the
 * stride are multiples of 32, so the reads of a slice's upper entries start on 256-byte boundaries. */
void acgb200_symdiag_layout(int nrows, const struct acgb200_symdiag *sd, int *margin, int *stride,
                            struct acgb200_symdiag_entry *tab)
{
    const int m = (sd->d[sd->nd - 1] + 31) & ~31;
    *margin = m;
    *stride = (m + nrows + 31) & ~31;
    for (int e = 0; e < sd->no; e++) {
        const int o = sd->o[e], a = o < 0 ? -o : o;
        int idx = 0;
        while (sd->d[idx] != a) idx++;
        tab[e].voff = idx * *stride + m + (o < 0 ? o : 0);
        tab[e].coff = o;
    }
}
