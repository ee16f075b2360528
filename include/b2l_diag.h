/* libb200diag.so -- micro-benchmarks used by tools/diag.py to size the kernels of libb200llama.
 * Debug only: nothing in the product library, the Python package, the tests or bench.py depends on it. */
#ifndef B2L_DIAG_H_
#define B2L_DIAG_H_
#include "b2l.h"
#ifdef __cplusplus
extern "C" {
#endif

const char* b2l_diag_last_error(void);

/* Debug only (tools/diag.py grid_flag): latency of a grid-wide arrive-and-wait on a global counter (red.release +
 * ld.acquire polling) with ctas_per_sm * SMs co-resident CTAs.  counter: zeroed device uint32; out: device
 * uint64[2 * rounds], first half zeroed (max ns per round), second half set to ~0 (min ns per round). */
int b2l_debug_grid_flag(void* out, void* counter, int ctas_per_sm, int rounds, b2l_stream_t stream);

/* Debug only (tools/diag.py hmma_rate): issue rate of mma.sync.m16n8k16 (f16, fp32 accumulate) on one SM:
 * one CTA of `warps` warps, `chains` (1, 2, 4, 8) independent accumulators per warp, iters x 8 MMAs per warp,
 * optionally preceded by the batch-1 kernel's 5 unpack ALU ops.  out: device uint64[2], out[0] = cycles. */
int b2l_debug_hmma_rate(void* out, int warps, int chains, int iters, int with_unpack, b2l_stream_t stream);

/* Debug only (tools/diag.py imma_rate): issue rate of mma.sync.m16n8k32 (u8 x s8, s32 accumulate) on one SM: one CTA
 * of `warps` warps, `chains` independent accumulators per warp, iters x 8 MMAs per warp, n_alu (0, 2, 4) ALU ops in
 * front of every MMA (2 = the two LOP3 of the int8 form of the int4 unpack).  out: device uint64[2], out[0] = cycles. */
int b2l_debug_imma_rate(void* out, int warps, int chains, int iters, int n_alu, b2l_stream_t stream);

/* Debug only (tools/diag.py consumer_rate): the decode kernels' consumer loop on stages already resident in shared
 * memory (no TMA, no barriers): cycles for `iters` sweeps over 8 stages of 16 KB.  mode bits: 1 weight LDS, 2 digit LDS,
 * 4 IMMA, 8 predicate the digit load of the unused lanes off.  out: device uint64[2], out[0] = cycles (CTA 0). */
int b2l_debug_consumer_rate(void* out, int warps, int iters, int mode, int n_ctas, b2l_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B2L_DIAG_H_ */
