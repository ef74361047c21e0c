/* eqf_b200_predict.h - C ABI of libeqf_b200_predict.so: the de-normalised OC20 IS2RE predictions of one batch.
 *
 *   energy_out[i] = energy[i] * std + mean                             for i < n_graphs
 *   pos_out[i, c] = pos[i, c] + (delta[i, c] * pos_std + 0.0f)         for i < n_rows with tags[i] > 0
 *   pos_out[i, c] = pos[i, c]                                          for i < n_rows with tags[i] <= 0
 *
 * The energy is ocpmodels' `Normalizer.denorm` (`tensor * std + mean`), the positions that of the positions normaliser
 * with mean 0 followed by `pred_pos[mask] + delta_pos[mask]` over the moving atoms (energy_trainer_v2.predict).  Each
 * operation is rounded on its own (no fused multiply-add), so the results are bitwise equal to the same float32 tensor
 * expressions run eagerly.  NaN and Inf propagate.  Rows at or past n_graphs / n_rows are not written.
 *
 * `energy` holds n_graphs or more floats (row i at energy[i]); `pos`, `delta` and `pos_out` are [n_rows, 3] row-major
 * floats and `tags` n_rows int64.  `delta == NULL` predicts the energies only, and then `pos`, `tags` and `pos_out` must be
 * NULL as well.  One launch, nothing read from the host and no synchronisation, so the call can be captured in a CUDA
 * graph.  Conventions as in eqf_b200.h: device pointers, `stream` is a cudaStream_t, 0 = ok, negative = error with a
 * message from eqf_last_error().
 */
#ifndef EQF_B200_PREDICT_H_
#define EQF_B200_PREDICT_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EQF_PREDICT_THREADS 256     /* threads per CTA, one row per thread and pass */
#define EQF_PREDICT_MAX_CTAS 128    /* grid cap: past 256 * 128 rows every CTA strides more than once */

const char* eqf_last_error(void);

int eqf_predict_is2re(const float* energy, int64_t n_graphs, float mean, float std, const float* pos, const float* delta,
                      const int64_t* tags, int64_t n_rows, float pos_std, float* energy_out, float* pos_out, void* stream);

/* The argument checks of eqf_predict_is2re on their own: host code only, nothing is launched or dereferenced.  The entry
 * point returns what this returns before it launches anything. */
int eqf_predict_is2re_check(const float* energy, int64_t n_graphs, const float* pos, const float* delta,
                            const int64_t* tags, int64_t n_rows, const float* energy_out, const float* pos_out);

#ifdef __cplusplus
}
#endif
#endif
