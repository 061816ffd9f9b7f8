/*
 * internal.h -- private interfaces between the C host layer and the CUDA
 * kernels of libacgb200.  Not installed; the public C-ABI is include/acgb200/.
 */
#ifndef ACGB200_INTERNAL_H
#define ACGB200_INTERNAL_H

#include <cuda_runtime_api.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------
 * SpMV tile plan
 *
 * The local CSR block is cut, once at init, into row-aligned tiles of at most
 * `rows_cap` rows and `nnz_cap` nonzeros.  A tile is one unit of TMA staging:
 * its slice of values / column indices / row pointers is fetched with three
 * cp.async.bulk copies into one shared-memory stage.  Bulk copies need
 * 16-byte aligned addresses and sizes, so every slice start is rounded down to
 * a multiple of 4 elements and every length rounded up; the device arrays are
 * allocated with padding so the over-read stays in bounds.
 *
 * Rows longer than nnz_cap ("long rows", power-law matrices) are left out of
 * the tiles and listed separately; a second kernel streams each of them with
 * several CTAs and combines partial sums with atomics.
 * ------------------------------------------------------------------------ */
struct acgb200_tile {        /* 16 bytes, read as one int4 */
    int row_begin;           /* first row of the tile */
    int nrows;               /* number of rows */
    int k_al;                /* rowptr[row_begin] rounded down to a multiple of 4 */
    int nnz_al;              /* padded slice length: multiple of 4, covers the tile's nonzeros */
};

#define ACGB200_SYMDIAG_MAX 64      /* = SLICE_MAXLEN (slices.c): entries per row of the mirrored-diagonal layout */
struct acgb200_symdiag_entry { int voff, coff; };   /* value offset (relative to the row), column offset */

struct acgb200_spmvplan {
    int nrows;                       /* rows covered (owned rows) */
    int64_t nnz;
    int lanes_per_row;               /* G: 1,2,4,8,16,32 */
    int rows_cap, nnz_cap;           /* tile limits */
    int nstages;                     /* smem ring depth */
    int threads;                     /* CTA size */
    int unroll;                      /* gathers in flight per lane */
    int ntiles;
    struct acgb200_tile *d_tiles;    /* [ntiles] */
    int nlong;                       /* rows with more than nnz_cap nonzeros */
    int *d_longrows;                 /* [nlong] */
    /* medium rows (opt-in, option "spmv_medium" = threshold): rows with more than med_thr and at most
     * nnz_cap nonzeros are left out of the tiles and get one warp each (spmv_medium_kernel); inside a
     * tile such a row would keep one G-lane group busy while the rest of the CTA idles */
    int med_thr;                     /* 0: off */
    int nmed;
    int *d_medrows;                  /* [nmed] */
    double *d_long_scratch;          /* [nlong * long_chunks] partial sums of the long-row kernels */
    int grid;                        /* persistent grid size */
    int smem_bytes;                  /* dynamic shared memory per CTA */
    int long_chunks;                 /* CTAs per long row */
    int max_ctas_per_sm;             /* 0: occupancy limit */
    /* pattern slices (slices.c): 32-row slices whose rows all repeat a dictionary pattern are stored
     * slice-major (entry e of the 32 rows contiguous, rows padded to the slice's longest) and multiplied by
     * spmv_slices_kernel -- 8 bytes per nonzero, no column indices, no row pointers, no shared-memory
     * staging; their rows are left out of the tiles */
    int nslices;
    struct acgb200_slice *d_slices;  /* [nslices] */
    double *d_sval;                  /* [sval_blocks * 32] */
    int64_t sval_blocks;             /* value blocks of 32 doubles (one per slice and entry slot) */
    int slice_rows;                  /* rows covered by slices */
    int64_t slice_nnz;               /* nonzeros covered (without padding) */
    int slice_lpad;                  /* row stride of the padded offset table */
    int slice_npat;
    int *d_spatoff;                  /* [slice_npat * slice_lpad] offsets col - row, zero beyond a pattern's length */
    unsigned short *d_spatid;        /* [nrows] pattern id per row (valid for covered rows) */
    int slice_ub, slice_threads, slice_grid, slice_smem, slice_max_ctas;
    int slice_ub_opt;                /* option "slice_ub" at init (0: slice_ub follows the row length, see slice_domlen) */
    int slice_domlen;                /* most frequent row length among covered rows (slice_ub without mirrored diagonals) */
    int64_t slice_exc, slice_excnnz; /* exception rows inside slices (columns from the CSR index array) and their nonzeros */
    /* mirrored diagonals (slices.c, acgb200_symdiag_plan): the slice-covered rows of a symmetric matrix read
     * their values from symdiag_nd stored upper diagonals, every lower entry from its mirror row
     * (spmv_symdiag_kernel instead of spmv_slices_kernel); 0: off.  Entry e of a covered row i is
     * d_hval[symdiag_tab[e].voff + i] times x[i + symdiag_tab[e].coff] (column clamped to [0, nrows)) */
    int symdiag_nd, symdiag_no;
    int symdiag_stride;              /* doubles per stored diagonal, the zero front margin included */
    struct acgb200_symdiag_entry symdiag_tab[ACGB200_SYMDIAG_MAX];
    int symdiag_d[ACGB200_SYMDIAG_MAX];   /* the stored diagonals D, ascending */
    int symdiag_margin;              /* zero entries in front of each diagonal (>= max D) */
    int symdiag_evict_first;         /* 1: stream the stored values with an L2 evict-first policy */
    double *d_hval;                  /* [symdiag_nd * symdiag_stride]; NULL once the coded layout replaced it */
    const int *symdiag_colidx;       /* device CSR columns the fill reads (borrowed, valid during init only) */
    int *d_symdiag_bad;              /* fill-time symmetry check: 0 passed (written by acgb200_slices_fill) */
    /* coded layout: when the stored diagonals hold at most 256 distinct bit patterns, one byte per element in
     * the same layout (d_hcode[voff + i] in place of d_hval[voff + i]) indexes a table of those doubles,
     * sorted by bit pattern.  Built and checked by acgb200_slices_fill when d_hcode and d_codes are set. */
    int symdiag_codes;               /* table entries; 0: the fp64 diagonals */
    int symdiag_try_codes;           /* option "symdiag_codes" at init: build the coded layout whenever the values allow */
    uint8_t *d_hcode;                /* [symdiag_nd * symdiag_stride] */
    struct acgb200_codestate *d_codes;   /* the table and the state of building it */
    int pcg_grid;                    /* grid of the fused pipelined-CG kernel (acgb200_pcg_fused_launch); 0: none */
    /* merge-path tiles (mergeplan.c): rows [0, merge_rows) of an irregular (power-law) matrix, cut into tiles
     * of merge_items merged items (row ends + nonzeros) and multiplied by spmv_merge_kernel; rows cut by tile
     * boundaries are finished by spmv_merge_fix_kernel from the tiles' partial sums */
    int nmtiles, nsplit, merge_items, merge_rows;
    int64_t merge_nnz;
    struct acgb200_mtile *d_mtiles;  /* [nmtiles] */
    struct acgb200_msplit *d_msplit; /* [nsplit] */
    double *d_mpart;                 /* [2 * nmtiles]: slot 0 head piece, slot 1 tail piece of each tile */
    int merge_grid, merge_smem, merge_threads, merge_stages, merge_max_ctas;
};

/* one merge-path tile: row ends of rows [r0, r0+nre), nonzeros [k0, k0+nnz) */
struct acgb200_mtile { int r0; int nre; int k0; int nnz; };
/* a row cut by tile boundaries: its pieces are the tail pieces of tiles ta..tb-1 and the head piece of tile tb */
struct acgb200_msplit { int row; int ta; int tb; int pad; };
struct acgb200_mergeplan {
    int ntiles, nsplit, items, rows;
    int64_t nnz;
    struct acgb200_mtile *tiles;
    struct acgb200_msplit *split;
};
int acgb200_merge_plan(int hi, const int64_t *rowptr, int items, struct acgb200_mergeplan *out);
void acgb200_mergeplan_free(struct acgb200_mergeplan *mp);

struct acgb200_patterns;

/* one covered slice: rows [row0, row0+32), `len` entry slots, values at d_sval + 32 * vblk */
struct acgb200_slice { int row0; int nrows; int len; int vblk; };

/* host plan of the pattern slices (no CUDA): which full 32-row slices of rows [0,cover_hi) are
 * covered, their descriptors, and the padded offset table.  Returns ACG_SUCCESS with *nslices == 0
 * when slices do not pay (few covered rows).  Arrays are malloc'ed, the caller frees them. */
struct acgb200_sliceplan {
    int nslices; struct acgb200_slice *slices;
    unsigned char *covered;          /* [(nrows+31)/32] 1: the slice's rows are handled by the slice kernel */
    int64_t blocks, nnz;
    int rows, lpad, npat, domlen;    /* domlen: most frequent row length among covered rows */
    int *spatoff;                    /* [npat * lpad] */
    unsigned short *patid;           /* [nrows] pattern id as the slice kernel sees it: < npat, or ACGB200_NOPATTERN =
                                      * exception row (columns from the index array) */
    int64_t nexc, excnnz;            /* exception rows inside covered slices, their nonzeros */
};
int acgb200_slices_plan(int nrows, int cover_hi, const int64_t *rowptr, const struct acgb200_patterns *pat,
                        struct acgb200_sliceplan *out);
void acgb200_sliceplan_free(struct acgb200_sliceplan *sp);

/* Mirrored diagonals of a slice plan (host, no CUDA).  O: the sorted union of the offsets col - row of the
 * covered rows; D = {|o| : o in O}, the diagonals stored.  Eligible (reason 0) if the plan has slices and no
 * exception rows, every covered row's offsets are strictly ascending, |O| <= ACGB200_SYMDIAG_MAX and 8|D|
 * bytes per covered row are fewer than the slice-major values they replace.  The values themselves are
 * checked on the device (acgb200_slices_fill). */
enum { SYMDIAG_OK = 0, SYMDIAG_NO_SLICES, SYMDIAG_EXCEPTIONS, SYMDIAG_UNSORTED, SYMDIAG_TOO_MANY, SYMDIAG_NO_GAIN,
       SYMDIAG_TOO_LARGE };
struct acgb200_symdiag {
    int reason;                      /* SYMDIAG_OK: eligible */
    int no, nd;
    int o[ACGB200_SYMDIAG_MAX];      /* O, ascending */
    int d[ACGB200_SYMDIAG_MAX];      /* D, ascending */
};
int acgb200_symdiag_plan(int nrows, const struct acgb200_sliceplan *sp, const struct acgb200_patterns *pat,
                         struct acgb200_symdiag *out);
/* the layout of an eligible plan: zero margin and stride of the diagonals, (value, column) offset per entry */
void acgb200_symdiag_layout(int nrows, const struct acgb200_symdiag *sd, int *margin, int *stride,
                            struct acgb200_symdiag_entry *tab);

/* Building the coded layout (kernels.cu): the distinct bit patterns of the stored diagonals go into an
 * open-addressing set, are sorted into vtab and every element is encoded, then decoded again and compared.
 * The host reads ncodes and bad once the fill has finished: 1 <= ncodes <= 256 and bad == 0 mean the codes
 * reproduce every stored double bit for bit. */
#define ACGB200_CODES_MAX 256
#define ACGB200_CODES_SET 1024       /* slots of the set; more than 256 patterns is an overflow before it fills */
struct acgb200_codestate {
    double vtab[ACGB200_CODES_MAX];  /* code c stands for vtab[c]; ascending by bit pattern */
    unsigned long long set[ACGB200_CODES_SET];   /* distinct patterns; all ones marks an empty slot ... */
    int has_ones;                    /* ... so that pattern itself (a NaN) is recorded here */
    int overflow;                    /* more than 256 distinct patterns */
    int ncodes;                      /* table entries; 0: no codes */
    int bad;                         /* 1: an element was not reproduced by its code */
};

/* fill d_sval from the device CSR values (kernels.cu); with pl->d_hval also the mirrored diagonals and
 * their symmetry check (pl->d_symdiag_bad), and with pl->d_hcode their codes (pl->d_codes) */
int acgb200_slices_fill(const struct acgb200_spmvplan *pl, const int *d_rowptr, const double *d_a, cudaStream_t stream);

/* row-pattern dictionary (compress.c): rows whose pattern id is not
 * ACGB200_NOPATTERN need no column indices, col = row + patoff[patptr[id] + j] */
#define ACGB200_NOPATTERN 0xFFFFu
struct acgb200_patterns {
    int npat, nentries;
    int *patptr;                 /* [npat+1] */
    int *patoff;                 /* [nentries] */
    unsigned short *patid;       /* [nrows] */
    int64_t nrows_matched;
};
int acgb200_patterns_build(int nrows, const int64_t *rowptr, const int *colidx, int max_entries,
                           struct acgb200_patterns *out);
void acgb200_patterns_free(struct acgb200_patterns *p);

/* epilogue of the SpMV kernels */
enum acgb200_spmvmode {
    SPMV_Y_AX = 0,        /* y = A x                                            */
    SPMV_Y_AX_DOT = 1,    /* y = A x ; acc += sum_{row<dotrows} x[row]*y[row]   */
    SPMV_R_B_AX = 2,      /* y = b - A x ; acc += sum_{row<dotrows} y[row]^2    */
    SPMV_Y_PLUS_AX = 3,   /* y += A x  (off-diagonal block)                     */
};

/* ------------------------------------------------------------------------
 * Device-resident CG state: iteration control and all scalars.  One
 * allocation; kernels never read a control word that the same kernel writes
 * (see DESIGN.md "control ring").
 * ------------------------------------------------------------------------ */
struct acgb200_ctrl { int iter; int done; int pad0, pad1; };

/* the largest group of iterations over which the fused pipelined CG defers its p and x updates */
#define ACGB200_PCG_GROUP_MAX 16

struct acgb200_devstate {
    struct acgb200_ctrl ctrl[4];     /* ring: kernel i of an iteration reads ctrl[i], writes ctrl[i+1 mod nk] */
    int maxits;
    int pad[3];
    double tol;                      /* stop when ||r|| < tol (0: never) */
    double final_rr;                 /* (r,r) at the iteration that set done */
    /* classic CG: slot = iteration parity */
    double pap_loc[2], pap[2];       /* local partial / global (p,Ap) */
    double rr_loc[2], rr[2];         /* (r_k,r_k) lives in slot k&1 */
    /* pipelined CG: {gamma,delta} = {(r,r),(w,r)}.  gd_loc is indexed by parity (slots 0, 1) on the two-kernel
     * path, and on the fused path as a ring of three: iteration k reads slot k%3, adds into (k+1)%3 and
     * zeroes (k+2)%3, so its last kernel never adds into a slot it zeroes (DESIGN.md section 4a) */
    double gd_loc[3][2], gd[2][2];
    double prev[2][2];               /* {gamma_{k-1}, alpha_{k-1}} read by update k from slot k&1 */
    /* the fused path's {alpha_k, beta_k}, written by update k into slot k % ACGB200_PCG_GROUP_MAX and read by
     * the catch-up update of k's group and by the finish (DESIGN.md section 4a) */
    double ab[ACGB200_PCG_GROUP_MAX][2];
    /* setup-time reductions */
    double tmp_loc[2], tmp[2];
    unsigned int ticket;             /* spare (last-CTA detection on one GPU) */
    unsigned int pad1;
};

/* ------------------------------------------------------------------------
 * Peer-memory exchange (NVLink 4 / NVSwitch, one process per GPU).
 *
 * Every rank exports one device allocation (the "window") through CUDA IPC:
 *
 *     uint64 hflag[MAXR]                halo sequence number, per sender rank
 *     uint64 rflag[NCH][MAXR]           reduction sequence number, per channel/rank
 *     double red[NCH][2][MAXR][2]       reduction partials [channel][parity][rank][2]
 *     double ghost[2][recvsize]         ghost values, double-buffered by parity
 *
 * Producers store straight into their peers' windows (remote stores over
 * NVLink) and then publish a sequence number with st.release.sys; consumers
 * spin with ld.acquire.sys on their own window.  This replaces, inside the CG
 * loop, the pack kernel + ncclSend/ncclRecv group + unpack of the halo exchange
 * (acg/halo.c:1456-1627) and the ncclAllReduce of 1-2 doubles
 * (acg/comm.c:371): see DESIGN.md section 6.
 * ------------------------------------------------------------------------ */
#define ACGB200_MAXR 64
#define ACGB200_NCH 2

struct acgb200_p2pdev {
    int nranks, rank;
    int nrecip, sendsize;                    /* halo send side: neighbours, entries */
    int sdispls[ACGB200_MAXR + 1];           /* my send segments */
    int peer_rdispl[ACGB200_MAXR];           /* where segment i starts in recipient i's ghost buffer */
    double *peer_ghost[ACGB200_MAXR][2];     /* recipient i's ghost buffers */
    unsigned long long *peer_hflag[ACGB200_MAXR];   /* recipient i's hflag slot for this rank */
    int nsenders;
    int senders[ACGB200_MAXR];               /* ranks this rank waits for */
    unsigned long long *my_hflag;            /* [MAXR] */
    double *my_ghost[2];
    double *peer_red[ACGB200_MAXR];          /* rank r's red[][][][] base */
    unsigned long long *peer_rflag[ACGB200_MAXR];   /* rank r's rflag[][] base */
    double *my_red;
    unsigned long long *my_rflag;
    unsigned long long hbase, rbase;         /* sequence bases of the current solve */
    unsigned long long timed_out;            /* set by a kernel whose wait for a peer exceeded timeout_ns; sticky
                                              * for the solve (hbase, rbase, timed_out are reset by one copy) */
    unsigned long long timeout_ns;           /* 0: wait for ever */
    unsigned int ticket;                     /* last-block detection (one kernel at a time uses it) */
    /* inverse send map: border row b (relative to borderrowoffset) is sent to
     * neighbours bq[e] at ghost offsets bdst[e], e in [bptr[b], bptr[b+1]) */
    int borderoff, nborder;
    const int *bptr, *bq, *bdst;
    int fuse;                                /* 1: producers push/publish themselves; 0: comm_post_kernel does */
};

/* After the producer of a vector / of reduction partials: push them to the
 * peers.  iter_override < 0: gated by *cin and using its iteration index. */
struct acgb200_postargs {
    struct acgb200_p2pdev *p2p;
    const struct acgb200_ctrl *cin;
    const struct acgb200_devstate *st;
    int iter_override;
    const double *vec; const int *sendbufidx;     /* halo part; vec == NULL: none */
    int ch; const double *redbase; int redstride, redcount, par_off, seq_off;   /* reduction part; ch < 0: none */
};
int acgb200_comm_post(const struct acgb200_postargs *a, cudaStream_t stream);

/* kernels.cu ------------------------------------------------------------- */

/* choose tile parameters for a matrix with the given shape; fills everything
 * in *plan except the device arrays */
void acgb200_spmv_choose(struct acgb200_spmvplan *plan, int nrows, int64_t nnz, int64_t maxrowlen);
int acgb200_spmv_configure(struct acgb200_spmvplan *plan);   /* occupancy -> grid; returns cudaError */

struct acgb200_spmvargs {
    const struct acgb200_spmvplan *plan;
    const int *rowptr;        /* [nrows+1] (+pad) */
    const int *colidx;        /* [nnz] (+pad) */
    const double *a;          /* [nnz] (+pad) */
    const double *x;
    double *y;
    const double *b;          /* SPMV_R_B_AX */
    double *acc;              /* device accumulator for the fused dot */
    int dotrows;              /* rows [0,dotrows) contribute to acc */
    int mode;
    const struct acgb200_ctrl *ctrl_in;   /* may be NULL: unconditional */
    struct acgb200_ctrl *ctrl_out;
    struct acgb200_devstate *st;          /* for per-iteration scalar housekeeping; may be NULL */
    int housekeeping;                     /* 0 none, 1 classic, 2 pipelined */
    /* peer-memory mode: the border x ghost block is applied inside the kernel
     * (ghost values from the window once the senders have published) and the
     * last CTA publishes the fused dot on reduction channel pub_ch */
    const struct acgb200_p2pdev *p2p;
    int od_rowoffset, od_nrows;
    const int *orowptr; const int *ocolidx; const double *oa;
    int pub_ch;                           /* -1: do not publish */
};
/* bytes one SpMV launch must move at least, given the plan (for reports) */
int64_t acgb200_spmv_min_bytes(const struct acgb200_spmvplan *plan);
int acgb200_spmv_launch(const struct acgb200_spmvargs *args, cudaStream_t stream);

/* y[rowoffset+i] (+)= sum_k oa[k]*x[xoffset + ocolidx[k]], i in [0,nrows): the
 * border x ghost block (acg/cgcuda.c:878); epilogue per `mode` */
struct acgb200_offdiagargs {
    int nrows;                /* border rows */
    int rowoffset;            /* borderrowoffset */
    const int *orowptr; const int *ocolidx; const double *oa;
    const double *x; double *y;
    double *acc; int mode;    /* SPMV_Y_PLUS_AX (+ dot with x over these rows if acc) or SPMV_R_B_AX-style minus */
    int minus;                /* y -= instead of += (residual) */
    int dotkind;              /* 0 none, 1 x[row]*y[row], 2 y[row]^2 */
    const struct acgb200_ctrl *ctrl_in;
    struct acgb200_ctrl *ctrl_out;
    struct acgb200_devstate *st;
    const struct acgb200_p2pdev *p2p;   /* not NULL: ghosts come from the peer-memory window */
    int p2p_iter_override;              /* >= 0: wait for that halo sequence index (setup) */
};
int acgb200_offdiag_launch(const struct acgb200_offdiagargs *args, cudaStream_t stream);

/* classic CG fused BLAS-1 (replace acg/cg-kernels-cuda.cu:119-303 and the two
 * cublasDdot calls at acg/cgcuda.c:894,933) */
/* p2p != NULL: reductions come from / go to the peer-memory window and the
 * kernels that produce the next SpMV input push its border entries themselves */
int acgb200_cg_update_r(int n, struct acgb200_devstate *st, int cin, int cout, int multi,
                        struct acgb200_p2pdev *p2p,
                        const double *t, double *r, cudaStream_t stream);
int acgb200_cg_update_xp(int n, struct acgb200_devstate *st, int cin, int cout, int multi,
                         struct acgb200_p2pdev *p2p,
                         const double *r, double *p, double *x, cudaStream_t stream);
/* pipelined CG fused update + next dots (replaces acg/cg-kernels-cuda.cu:187-269
 * and the cublasDdot calls at acg/cgcuda.c:1680,1688) */
int acgb200_pcg_update(int n, struct acgb200_devstate *st, int cin, int cout, int multi,
                       struct acgb200_p2pdev *p2p,
                       const double *q, double *z, double *w, double *t, double *p,
                       double *r, double *x, cudaStream_t stream);

/* One whole pipelined-CG iteration on one GPU for a plan with mirrored diagonals and no merge tiles, medium
 * or long rows: the covered rows' product and update in one kernel (spmv_symdiag_kernel with its PCG
 * epilogue), which reads the control word ctrl[cin] and writes ctrl[cin ^ 1].  With tiles, the tile kernel
 * (q = A w over the other rows) and their update run first and pass the word through ctrl[2] and ctrl[3].
 * w is read, w_{k+1} goes to w_next (another buffer: other rows still gather w); z, t in place.  r_j lives
 * in slot j % group of a ring: slot 0 is the solver's r, slot s > 0 is r_ring + (s - 1) r_stride.  r_k is
 * read from r, slot k % group, and r_{k+1} goes to r_next, slot (k+1) % group.  p and x are updated by the
 * catch-up iteration only, the last of each group, for the whole group (DESIGN.md section 4a). */
struct acgb200_pcgargs {
    const struct acgb200_spmvplan *plan;
    const int *rowptr, *colidx; const double *a;    /* CSR of the tile rows */
    const double *w; double *w_next;
    double *q;                                      /* the tile rows' product */
    double *z, *t, *p, *r, *r_next, *x;
    const double *r_ring; size_t r_stride;          /* slots 1 ... group - 1 of the r ring */
    int group;                                      /* iterations per group, even, 2 ... ACGB200_PCG_GROUP_MAX */
    int catchup;                                    /* 1: k % group == group - 1 */
    struct acgb200_devstate *st;
    int cin;                                        /* 0 or 1: the iteration's parity */
    int vec_evict_first;                            /* L2 policy of the fused kernel's vector streams */
};
/* Weak in the host code, like the multi-vector launchers below: the host-logic test build of tests/hostsim
 * never plans mirrored diagonals, so it never selects this path and need not define it. */
#if defined(__CUDACC__)
#define ACGB200_MULTI_LAUNCHER
#else
#define ACGB200_MULTI_LAUNCHER __attribute__((weak))
#endif
ACGB200_MULTI_LAUNCHER int acgb200_pcg_fused_launch(const struct acgb200_pcgargs *a, cudaStream_t stream);
/* After the fused loop, whose final control word is ctrl[cfin]: if the updates done are not a multiple of
 * the group, the p and x updates of the last, partial group, and the last r moved from its ring slot into r;
 * otherwise nothing.  Leaves p, x and r as the plain recurrence does. */
ACGB200_MULTI_LAUNCHER int acgb200_pcg_fused_finish(int n, const struct acgb200_devstate *st, int cfin, int group,
                                                    double *r, const double *r_ring, size_t r_stride, double *p,
                                                    double *x, cudaStream_t stream);
/* the bytes the plain recurrence's fused launch moves (|D| elements + 96 per covered row), and those of a
 * whole fused iteration, averaged over a group of `group` iterations (the tile kernel's product, then per
 * row of the update 64 + (32 + 8 group) / group bytes in the slices and 8 more in the tiles, DESIGN.md
 * section 4a) */
int64_t acgb200_pcg_fused_min_bytes(const struct acgb200_spmvplan *plan);
int64_t acgb200_pcg_iteration_min_bytes(const struct acgb200_spmvplan *plan, int group);

/* the reference's public BLAS-1 building blocks (acg/cg-kernels-cuda.h:45-97; cgcuda.c wraps them) */
int acgb200_helper_axpy(int op, int n, const double *num, const double *den, const double *x, double *y, cudaStream_t stream);
int acgb200_helper_scalars(int op, double *out0, double *out1, const double *num, const double *den, cudaStream_t stream);
int acgb200_helper_pipelined(int n, const double *gamma, double *gamma_prev, const double *delta, const double *q,
                             double *p, double *r, double *t, double *x, double *z, double *w, double *alpha_prev,
                             cudaStream_t stream);

/* expand.cu: full-storage expansion of the packed symmetric CSR on the device
 * (the GPU form of acgsymcsrmatrix_dsymv_init, acg/symcsrmatrix.c:760-851) */
struct acgb200_expanded {
    int *d_rowptr; int *d_colidx; double *d_a;          /* local block, 0-based columns */
    int *d_orowptr; int *d_ocolidx; double *d_oa;       /* border x ghost block, columns rebased by -borderrowoffset */
    int64_t fnnz, onnz;
};
int acgb200_expand_device(int n, int ghost0, int border0, int nob, int64_t pnnz,
                          const int *d_prp, const int *d_pcol, const double *d_pa, double eps,
                          int rp_pad, int blk_pad, struct acgb200_expanded *out, cudaStream_t stream);

struct acgsymcsrmatrix;
/* expand_host.c: upload the packed matrix and expand it on the device (rp_pad / blk_pad: trailing
 * padding of the row-pointer / column+value arrays, as the TMA tile copies need) */
int acgb200_expand_upload(const struct acgsymcsrmatrix *A, double eps, int rp_pad, int blk_pad,
                          struct acgb200_expanded *out, cudaStream_t stream, int *errcode);
void acgb200_expanded_free(struct acgb200_expanded *x);

/* ------------------------------------------------------------------------
 * Several right-hand sides (acgsolvercuda_solve_multi): K independent classic
 * CG recurrences that share every pass over the matrix.  Block vectors hold K
 * columns interleaved, entry (row, j) at row*K + j, K in {1,2,4,8}.  Columns
 * beyond the caller's count are padding, inactive from the start.  The
 * active-column mask travels with the control word (ctrl.pad0, bit j), so it
 * follows the same ring as the iteration index.
 * ------------------------------------------------------------------------ */
#define ACGB200_MAXK 8

struct acgb200_mstate {
    double rr[2][ACGB200_MAXK];      /* (r_j,r_j) of iteration k in slot k&1 */
    double pap[2][ACGB200_MAXK];     /* (p_j,A p_j) of iteration k in slot k&1 */
    double tol[ACGB200_MAXK];        /* stop column j when ||r_j|| < tol[j] (0: never) */
    double final_rr[ACGB200_MAXK];   /* (r_j,r_j) of the column's last iterate */
    double tmp[ACGB200_MAXK];        /* set-up reductions */
    int nits[ACGB200_MAXK];          /* iterations the column ran */
    int conv[ACGB200_MAXK];          /* 1: the column met its tolerance */
};

struct acgb200_spmmargs {
    const struct acgb200_spmvplan *plan;  /* pattern slices of the single-vector plan */
    int k;                                /* block width K */
    int nranges;                          /* row chunks outside the slices, spmm_rows_kernel */
    const int *ranges;                    /* [2 * nranges]: first row, one past the last row */
    int lanes;                            /* lanes per row of spmm_rows_kernel: 1 or 8 */
    const int *rowptr, *colidx;
    const double *a;
    const double *x;                      /* n x K */
    double *y;                            /* n x K */
    const double *b;                      /* n x K, SPMV_R_B_AX */
    double *acc;                          /* [K] fused per-column dots (modes 1, 2); may be NULL */
    int mode;                             /* SPMV_Y_AX, SPMV_Y_AX_DOT or SPMV_R_B_AX */
    const struct acgb200_ctrl *ctrl_in;   /* may be NULL: unconditional */
    struct acgb200_ctrl *ctrl_out;
    const struct acgb200_devstate *st;    /* maxits of the gate */
    struct acgb200_mstate *ms;            /* housekeeping: the first kernel zeroes ms->rr[s^1] (may be NULL) */
};
/* The host code (cgcuda.c) references the four multi-vector launchers weakly: a host build that carries the
 * single-vector kernels only -- the host-logic test build of tests/hostsim -- still loads, and
 * acgsolvercuda_solve_multi / acgsolvercuda_spmm_mode return ACG_ERR_NOT_SUPPORTED there (no other path
 * runs instead).  libacgb200.so always defines them (kernels.cu). */
ACGB200_MULTI_LAUNCHER int acgb200_spmm_launch(const struct acgb200_spmmargs *a, cudaStream_t stream);
/* classic CG updates with per-column alpha_j, beta_j; columns outside the incoming mask are left alone */
ACGB200_MULTI_LAUNCHER int acgb200_cg_multi_update_r(int n, int k, struct acgb200_devstate *st, struct acgb200_mstate *ms, int cin, int cout,
                              const double *t, double *r, cudaStream_t stream);
ACGB200_MULTI_LAUNCHER int acgb200_cg_multi_update_xp(int n, int k, struct acgb200_devstate *st, struct acgb200_mstate *ms, int cin, int cout,
                               const double *r, double *p, double *x, cudaStream_t stream);
/* acc[j] += sum_i x[i*k + j]^2 */
ACGB200_MULTI_LAUNCHER int acgb200_dot_multi(int n, int k, const double *x, double *acc, cudaStream_t stream);

/* ------------------------------------------------------------------------
 * Shifted systems (acgsolvercuda_solve_shifted): one seed CG on A drives
 * (A + sigma_j I) x_j = b for K shifts (multi-shift CG).  The seed runs the
 * single-vector classic loop on d_r, d_p, d_t; X_j and P_j live in block
 * vectors of width K (d_mx, d_mp), with the same padding and active-column
 * mask (ctrl.pad0) as the multi-vector loop.  Per-shift scalars are
 * double-buffered by iteration parity: iteration k reads slot k&1 and block 0
 * of its update writes slot (k&1)^1, so no kernel reads a slot it writes.
 * ------------------------------------------------------------------------ */
struct acgb200_sstate {
    double zeta[2][ACGB200_MAXK];       /* zeta_k of shift j in slot k&1 (zeta_0 = 1) */
    double zeta_prev[2][ACGB200_MAXK];  /* zeta_{k-1} in slot k&1 (zeta_{-1} = 1) */
    double ab_prev[2][2];               /* the seed's {alpha_{k-1}, beta_{k-1}} in slot k&1 ({1, 0} at k = 0) */
    double sigma[ACGB200_MAXK];         /* the shifts */
    double tol[ACGB200_MAXK];           /* stop shift j when |zeta_j| ||r|| < tol[j] (0: never) */
    double final_rnrm2[ACGB200_MAXK];   /* |zeta_j| ||r|| of the shift's last iterate */
    int nits[ACGB200_MAXK];             /* iterations the shift ran */
    int conv[ACGB200_MAXK];             /* 1: the shift met its tolerance */
};
/* set-up: r = p = b, X_j = 0 and P_j = b for all k columns */
ACGB200_MULTI_LAUNCHER int acgb200_shift_setup(int n, int k, const double *b, double *r, double *p, double *x, double *pk,
                                               cudaStream_t stream);
/* after acgb200_cg_update_r: the seed's p = r + beta p, and for each active shift X_j += alpha_j P_j ;
 * P_j = zeta_{k+1,j} r + beta_j P_j.  Block 0 advances the control word, applies each shift's
 * convergence test and clears the next product's (p,Ap) accumulator. */
ACGB200_MULTI_LAUNCHER int acgb200_cg_shift_update(int n, int k, struct acgb200_devstate *st, struct acgb200_sstate *ss,
                                                   int cin, int cout, const double *r, double *p, double *x, double *pk,
                                                   cudaStream_t stream);

/* ------------------------------------------------------------------------
 * MINRES (acgsolvercuda_solve_minres): unpreconditioned Paige-Saunders on the
 * single-vector product, for symmetric A that may be indefinite.  Iteration k
 * (parity s = k&1) runs the product t = A v_k with alpha_k = (v_k, t) into
 * alpha[s], the Lanczos kernel (u = t - alpha_k v_k - beta_k v_{k-1} in place
 * in t, (u,u) into uu[s]) and the update kernel (Givens rotation, w_k, x,
 * v_{k+1}).  v_{k+1} overwrites v_{k-1} and w_k overwrites w_{k-2}: two buffers
 * each, chosen by parity.  The scalars of iteration k are read from slot s;
 * block 0 of the update writes slot s^1 and zeroes alpha[s^1] and uu[s^1], so
 * no kernel reads a slot it writes.
 * ------------------------------------------------------------------------ */
struct acgb200_nstate {
    double alpha[2];                 /* (v_k, A v_k), accumulated by the product */
    double uu[2];                    /* (u, u) = beta_{k+1}^2, accumulated by the Lanczos kernel */
    double beta[2];                  /* beta_k */
    double cs[2], sn[2];             /* the previous rotation c_{k-1}, s_{k-1} */
    double dbar[2], eps[2];          /* delta-bar_k, epsilon_k */
    double phibar[2];                /* phi-bar_k: the recursively updated residual norm */
};
/* set-up: v *= scale (v_1 = r_0 / beta_1), vprev = w0 = w1 = 0 */
ACGB200_MULTI_LAUNCHER int acgb200_minres_setup(int n, double scale, double *v, double *vprev, double *w0, double *w1,
                                                cudaStream_t stream);
/* u = t - alpha_k v - beta_k vprev in place in t, (u,u) into ns->uu[k&1]; reads the control word ctrl[cin] */
ACGB200_MULTI_LAUNCHER int acgb200_minres_lanczos(int n, const struct acgb200_devstate *st, struct acgb200_nstate *ns,
                                                  int cin, const double *v, const double *vprev, double *t,
                                                  cudaStream_t stream);
/* The rotation from slot k&1 and beta_{k+1} = sqrt(uu), then w_k = (v - eps_k w_{k-2} - delta_k w_{k-1}) / gamma_k
 * into w (which holds w_{k-2}), x += phi_k w_k, vnext = u / beta_{k+1}.  Block 0 writes slot (k&1)^1, ends the
 * loop on phi-bar_{k+1} < tol or beta_{k+1} = 0 (after the update) or gamma_k = 0 (before it, the iteration not
 * counted), zeroes the next accumulators and writes ctrl[cout]. */
ACGB200_MULTI_LAUNCHER int acgb200_minres_update(int n, struct acgb200_devstate *st, struct acgb200_nstate *ns,
                                                 int cin, int cout, const double *v, const double *u, double *w,
                                                 const double *wprev, double *x, double *vnext, cudaStream_t stream);

/* ------------------------------------------------------------------------
 * Mixed-precision CG with reliable updates (acgsolvercuda_solve_mixed): r, p,
 * t and y are float vectors scaled by an exact power of two sigma; every
 * operation is fp64 and each stored value is rounded once.  x and b stay fp64.
 * Iteration k (parity s = k&1) runs five steps:
 *   1. t = fl32(A p), pi = (p, t) into pi[s]                 reads ctrl[0]
 *   2. r = fl32(r - alpha t), (r,r) into rr[s]               reads ctrl[0]
 *   3. y = fl32(y + alpha p); not due: p = fl32(r + beta p); due: x += sigma y,
 *      y = 0.  Block 0 writes ctrl[1] (the word after the iteration when no
 *      update is due) and ctrl[2] (active only when one is due)  reads ctrl[0]
 *   4. r64 = b - A x with (r64,r64) into rr64[s]: the fp64 product, gated by
 *      ctrl[2] (its tile kernel copies the word into ctrl[3], read by nobody)
 *   5. the replacement: rescale r and p from r64, the convergence test, and
 *      ctrl[0] for the next iteration (ctrl[1] when no update was due)
 * Slot s holds the scalars iteration k reads; block 0 of step 3 or 5 writes
 * slot s^1 and zeroes its accumulators, so no kernel reads a slot it writes.
 * ------------------------------------------------------------------------ */
struct acgb200_xstate {
    double pi[2];                    /* (p, A p) of the fp32 product */
    double rr[2];                    /* rho' = (r, r) after update_r */
    double rr64[2];                  /* (r64, r64) of a reliable update's fp64 residual */
    double rho[2];                   /* rho_k = (r_k, r_k), scaled by 1/sigma^2 */
    double mx[2];                    /* M: the largest sqrt(rho) since the last reliable update */
    double sigma[2];                 /* the scale of the fp32 vectors (a power of two) */
    double last_rr64;                /* (r64, r64) of the x of the last fold (x0 at set-up) */
    int nupdates;                    /* reliable updates of the solve */
    int conv;                        /* 1: a reliable update met the tolerance (or r64 = 0) */
    int breakdown;                   /* 1: pi = 0 or non-finite ended the solve */
    int pad;
};
/* the product t = fl32(A p) on float vectors: mirrored-diagonal rows through spmv_symdiag_kernel (float
 * gathers and store), every other row through a CSR rows kernel over `ranges`, one thread per row in CSR
 * order; acc += (p, t) over all rows if acc.  ctrl_in may be NULL (ungated). */
struct acgb200_spmvf32args {
    const struct acgb200_spmvplan *plan;  /* its mirrored diagonals, if symdiag_nd > 0 */
    int nranges;                          /* row chunks the diagonals do not cover */
    const int *ranges;                    /* [2 * nranges]: first row, one past the last row */
    const int *rowptr, *colidx;
    const double *a;
    const float *x;
    float *y;
    double *acc;
    const struct acgb200_ctrl *ctrl_in;
    const struct acgb200_devstate *st;
};
ACGB200_MULTI_LAUNCHER int acgb200_spmv_f32_launch(const struct acgb200_spmvf32args *a, cudaStream_t stream);
/* set-up: r = fl32(r64 * scale), p = r, y = 0 (scale = 1/sigma) */
ACGB200_MULTI_LAUNCHER int acgb200_mixed_setup(int n, double scale, const double *r64, float *r, float *p, float *y,
                                               cudaStream_t stream);
/* step 2 (reads ctrl[0]) */
ACGB200_MULTI_LAUNCHER int acgb200_mixed_update_r(int n, const struct acgb200_devstate *st, struct acgb200_xstate *xs,
                                                  const float *t, float *r, cudaStream_t stream);
/* step 3 (reads ctrl[0], writes ctrl[1] and ctrl[2]) */
ACGB200_MULTI_LAUNCHER int acgb200_mixed_update_yp(int n, struct acgb200_devstate *st, struct acgb200_xstate *xs,
                                                   const float *r, float *p, float *y, double *x, cudaStream_t stream);
/* step 5 (reads ctrl[1] and ctrl[2], writes ctrl[0]) */
ACGB200_MULTI_LAUNCHER int acgb200_mixed_replace(int n, struct acgb200_devstate *st, struct acgb200_xstate *xs,
                                                 const double *r64, float *r, float *p, cudaStream_t stream);
/* x += sigma y (the fold at maxits; ungated) */
ACGB200_MULTI_LAUNCHER int acgb200_mixed_fold(int n, double sigma, const float *y, double *x, cudaStream_t stream);

/* ------------------------------------------------------------------------
 * Chebyshev-preconditioned CG (acgsolvercuda_solve_chebyshev): PCG with
 * M^-1 = p_d(D^-1 A) D^-1, z = M^-1 r formed by d steps of Jacobi-scaled
 * Chebyshev iteration on A z = r from z = 0 (DESIGN.md section 15).
 * Iteration k (parity s = k&1) runs:
 *   1. t = A p with (p, t) into pap[s]                        reads ctrl[0]
 *   2. the r/x kernel: alpha = rz[k%3]/pap[s], x += alpha p, r -= alpha t,
 *      (r, r) into rr[s], and the preconditioner's start (degree 0: z = D^-1 r
 *      with (r, z) into rz[(k+1)%3])            reads ctrl[1], writes ctrl[2]
 *   3. d inner steps res -= A d_{j-1}, d_j = c1_j d_{j-1} + c2_j D^-1 res,
 *      z += d_j; the last adds (r, z) into rz[(k+1)%3]          read ctrl[2]
 *   4. the p kernel: the test on (r, r), p = z + beta p      reads ctrl[2],
 *      writes ctrl[0]
 * (r, z) lives in a ring of three slots: the p kernel of iteration k reads
 * slots k%3 and (k+1)%3 and zeroes (k+2)%3, so no kernel reads a slot it
 * writes.  The set-up's preconditioner is that of "iteration -1": it adds into
 * slot 0.
 * ------------------------------------------------------------------------ */
#define ACGB200_CHEB_MAXDEG 16
#define ACGB200_CHEB_EST 10             /* Jacobi-PCG steps of the interval estimate */
struct acgb200_cstate {
    double pap[2];                   /* (p, A p) of iteration k in slot k&1 */
    double rr[2];                    /* (r_{k+1}, r_{k+1}) of iteration k in slot k&1 */
    double rz[3];                    /* (r_k, z_k) in slot k%3 */
    double alpha_log[ACGB200_CHEB_EST], beta_log[ACGB200_CHEB_EST];   /* the estimate's alpha_k, beta_k */
    int log;                         /* 1: log alpha_k and beta_k (the estimate) */
    int breakdown;                   /* 1: (p, A p) or (r, z) <= 0 or non-finite ended the solve */
    int baddiag;                     /* diagonal entries <= 0 or non-finite (acgb200_cheb_dinv) */
    int pad;
};
/* dinv_i = 1 / a_ii of the full-storage local block; cs->baddiag += entries that are <= 0, non-finite or absent */
ACGB200_MULTI_LAUNCHER int acgb200_cheb_dinv(int n, const int *rowptr, const int *colidx, const double *a, double *dinv,
                                             struct acgb200_cstate *cs, cudaStream_t stream);
/* step 2 (reads ctrl[1], writes ctrl[2]).  start: the set-up's preconditioner start only (no breakdown test,
 * no update of x and r); x == NULL: x is not updated (the estimate).  cheb: res = r, d0 = c0 D^-1 r, z = d0;
 * otherwise z = D^-1 r with (r, z) folded in. */
ACGB200_MULTI_LAUNCHER int acgb200_cheb_rx(int n, struct acgb200_devstate *st, struct acgb200_cstate *cs, int start,
                                           int cheb, double c0, const double *dinv, const double *t, const double *p,
                                           double *x, double *r, double *z, double *res, double *d0,
                                           cudaStream_t stream);
/* step 3 on plans without the fused path: after q = A dprev, res -= q, dnext = c1 dprev + c2 D^-1 res,
 * z += dnext; last: (r, z) folded in, res and dnext not stored (reads ctrl[2]) */
ACGB200_MULTI_LAUNCHER int acgb200_cheb_step(int n, const struct acgb200_devstate *st, struct acgb200_cstate *cs, double c1,
                                             double c2, int last, const double *q, const double *dinv,
                                             const double *dprev, double *dnext, double *res, double *z,
                                             const double *r, cudaStream_t stream);
/* step 3 in one kernel per step (two with tiles) on plans with mirrored diagonals and no merge tiles, medium
 * or long rows: the mirrored-diagonal product of dprev goes straight into the step; the tile rows' product
 * goes to q first and is finished by the same kernel */
struct acgb200_chebargs {
    const struct acgb200_spmvplan *plan;
    const int *rowptr, *colidx; const double *a;    /* CSR of the tile rows */
    const struct acgb200_devstate *st;
    struct acgb200_cstate *cs;
    double c1, c2;
    int last;
    double *q;                                      /* the tile rows' product */
    const double *dinv, *dprev;
    double *dnext, *res, *z;
    const double *r;
};
ACGB200_MULTI_LAUNCHER int acgb200_cheb_fused_step(const struct acgb200_chebargs *a, cudaStream_t stream);
/* step 4 (reads ctrl[2], writes ctrl[0]) */
ACGB200_MULTI_LAUNCHER int acgb200_cheb_p(int n, struct acgb200_devstate *st, struct acgb200_cstate *cs,
                                          const double *z, double *p, cudaStream_t stream);

/* setup-time helpers */
int acgb200_dot(int n, const double *x, const double *y, double *acc, cudaStream_t stream); /* acc += x.y */
int acgb200_dot2(int n, const double *r, const double *w, double *acc2, cudaStream_t stream); /* acc2[0]+=r.r, acc2[1]+=w.r */
int acgb200_gather(int n, double *dst, const double *src, const int *idx, cudaStream_t stream);  /* dst[i]=src[idx[i]] */
int acgb200_scatter(int n, const double *src, double *dst, const int *idx, cudaStream_t stream); /* dst[idx[i]]=src[i] */
/* *first = min(*first, the smallest k < n with a[k] != b[k]): set *first to all ones before the first call, and
 * it still holds all ones afterwards exactly when the arrays agree.  Weak in the host code like the launchers
 * above: a host-logic test build without it refuses acgsolvercuda_update_values. */
ACGB200_MULTI_LAUNCHER int acgb200_first_diff(int64_t n, const int *a, const int *b, unsigned long long *first,
                                              cudaStream_t stream);
int acgb200_num_sms(void);
void acgb200_blas1_set_ctas_per_sm(int v);
void acgb200_set_pdl(int v);

#ifdef __cplusplus
}
#endif
#endif
