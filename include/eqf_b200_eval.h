/* eqf_b200_eval.h - C ABI of libeqf_b200_eval.so: the metric terms of an evaluation pass, added to a running accumulator.
 *
 * The accumulator is a small float64 array of slots on the device.  Each call adds one batch's terms to the slots it owns
 * (`acc` points at the first of them).  Every term is formed in float32 from the model's outputs, in the operation order
 * of the reference's expression and with no fused multiply-add, then widened to double and summed:
 *
 *   eqf_eval_graph  (EQF_EVAL_GRAPH_SLOTS, rows i < n_graphs; e = pred[i] * std + mean - y[i]):
 *                   acc[0] += sum |e|,  acc[1] += sum e * e,  acc[2] += #{|e| < threshold},
 *                   acc[3] += sum |pred[i] - (y[i] - mean) / std|,  acc[4] += n_graphs
 *   eqf_eval_atom   (EQF_EVAL_ATOM_SLOTS, rows i < n = min(max(*n_atoms, 0), n_rows) of the [n_rows, 3] arrays):
 *                   acc[0] += sum over components |pred_dy * std - dy|,
 *                   acc[1] += sum over atoms ||pred_dy - dy / std||_2 (the norm in float32),  acc[2] += n
 *   eqf_eval_batch  (EQF_EVAL_BATCH_SLOTS):  acc[0] += *loss (nothing when loss is NULL),  acc[1] += 1
 *
 * NaN and Inf propagate into the sums; a NaN error is not within the threshold.  The real atom count `n_atoms` is read on
 * the device, so nothing is read from the host and the calls can be captured in a CUDA graph.  The sums are fixed-order
 * reductions: one double partial per CTA and term, summed in CTA order by the CTA that finishes last, so repeated passes
 * are bitwise equal.  `partials` is caller-owned scratch of EQF_EVAL_SCRATCH doubles and `tickets` an int32 counter,
 * zero before the first call; each call leaves it at zero.  Calls on one stream may share both.  Conventions as in
 * eqf_b200.h: device pointers, `stream` is a cudaStream_t, 0 = ok, negative = error with a message from eqf_last_error().
 */
#ifndef EQF_B200_EVAL_H_
#define EQF_B200_EVAL_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EQF_EVAL_THREADS 256      /* threads per CTA, one row per thread and pass */
#define EQF_EVAL_MAX_CTAS 128     /* grid cap: past 256 * 128 rows every CTA strides more than once */
#define EQF_EVAL_MAX_TERMS 4      /* summed terms per call (the count is not one) */
#define EQF_EVAL_SCRATCH 512      /* EQF_EVAL_MAX_CTAS * EQF_EVAL_MAX_TERMS: doubles of the partials scratch */
#define EQF_EVAL_GRAPH_SLOTS 5
#define EQF_EVAL_ATOM_SLOTS 3
#define EQF_EVAL_BATCH_SLOTS 2

const char* eqf_last_error(void);

/* pred: n_graphs or more floats (row i at pred[i], the normalised output), y: n_graphs floats */
int eqf_eval_graph(const float* pred, const float* y, int64_t n_graphs, float mean, float std, float threshold,
                   double* partials, int32_t* tickets, double* acc, void* stream);

/* pred_dy, dy: [n_rows, 3] row-major floats; n_atoms: one int64 on the device, the real rows (the rest is padding) */
int eqf_eval_atom(const float* pred_dy, const float* dy, int64_t n_rows, const int64_t* n_atoms, float std,
                  double* partials, int32_t* tickets, double* acc, void* stream);

/* loss: one float on the device, or NULL to count the batch only */
int eqf_eval_batch(const float* loss, double* acc, void* stream);

/* The argument checks of the three entry points on their own: host code only, nothing is launched or dereferenced.
 * Each entry point returns what its check returns before it launches anything. */
int eqf_eval_graph_check(const float* pred, const float* y, int64_t n_graphs, const double* partials,
                         const int32_t* tickets, const double* acc);
int eqf_eval_atom_check(const float* pred_dy, const float* dy, int64_t n_rows, const int64_t* n_atoms,
                        const double* partials, const int32_t* tickets, const double* acc);
int eqf_eval_batch_check(const float* loss, const double* acc);

#ifdef __cplusplus
}
#endif
#endif
