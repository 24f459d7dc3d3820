/*
 * ORACLE — TEST INFRASTRUCTURE ONLY (see zuko_oracle_impl.h for the contract).
 * Builds the fp32 (_f32) and fp64 (_f64) variants of the CPU restatement.
 *   gcc -O3 -mavx2 -mfma -fopenmp -shared -fPIC zuko_oracle.c -o libzuko_oracle.so -lm
 * No -ffast-math: the fp32 variant must round like the reference's eager ops.
 */
#include <math.h>
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>

#define ZO_MAX_BINS 1024 /* the engine's RQS limit (bins in [1, 1024]); the knot arrays live on the stack */

#define REAL float
#define SUFFIX _f32
#define R_ABS fabsf
#define R_EXP expf
#define R_LOG logf
#define R_LOG1P log1pf
#define R_SQRT sqrtf
#include "zuko_oracle_impl.h"
#undef REAL
#undef SUFFIX
#undef R_ABS
#undef R_EXP
#undef R_LOG
#undef R_LOG1P
#undef R_SQRT

#define REAL double
#define SUFFIX _f64
#define R_ABS fabs
#define R_EXP exp
#define R_LOG log
#define R_LOG1P log1p
#define R_SQRT sqrt
#include "zuko_oracle_impl.h"

int zo_max_bins(void) { return ZO_MAX_BINS; }

#ifdef _OPENMP
#include <omp.h>
/* torchrun exports OMP_NUM_THREADS=1; the CPU baseline sets its thread count explicitly. */
void zo_set_threads(int n) { if (n > 0) omp_set_num_threads(n); }
int zo_get_threads(void) { return omp_get_max_threads(); }
#else
void zo_set_threads(int n) { (void)n; }
int zo_get_threads(void) { return 1; }
#endif
