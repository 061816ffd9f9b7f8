/*
 * kernels_refresh_sim.c -- TEST INFRASTRUCTURE ONLY.  Plain-C stand-in for the structure comparison of
 * acgsolvercuda_update_values (acgb200_first_diff, kernels.cu): the first index at which two "device" int
 * arrays differ, folded into *first as the kernel's atomicMin does.
 */
#include "internal.h"
#include "hostsim.h"

int acgb200_first_diff(int64_t n, const int *a, const int *b, unsigned long long *first, cudaStream_t stream)
{
    (void) stream;
    for (int64_t k = 0; k < n; k++)
        if (a[k] != b[k]) { if ((unsigned long long) k < *first) *first = (unsigned long long) k; break; }
    return 0;
}
