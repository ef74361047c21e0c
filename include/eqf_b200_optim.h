/* eqf_b200_optim.h - C ABI of libeqf_b200_optim.so: gradient-norm clipping, AdamW and the model EMA on flat buffers.
 *
 * Every buffer is one fp32 array of n elements (the flat parameter / gradient buckets of equiformer_b200.parallel),
 * 16-byte aligned; n need not be a multiple of 4.  The scalars that change from step to step (the clip coefficient, the
 * learning rate and the step count) live in device memory, so neither entry point reads anything from the host and a
 * step can be captured in a CUDA graph and replayed.
 *
 *   eqf_flat_sqnorm:  norm = ||g||_2 (squares summed in double),  coef = min(1, max_norm / (norm + 1e-6))
 *                     as torch.nn.utils.clip_grad_norm_ computes it: a NaN or Inf norm gives a NaN or 0 coefficient.
 *   eqf_flat_adamw:   t += 1;  g *= coef;  m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;
 *                     p -= lr * decay[i] * p;  p -= lr / (1-b1^t) * m / (sqrt(v) / sqrt(1-b2^t) + eps);
 *                     ema += (1-ema_decay) (p - ema)   (when ema is given)
 *
 * The sums of squares are fixed-order reductions: one partial per CTA (in double), summed in CTA order by the CTA that
 * finishes last, so runs are bitwise reproducible.  `tickets` is a caller-owned int32 counter, zero before the first
 * call; each kernel leaves it at zero.  Conventions as in eqf_b200.h: device pointers, `stream` is a cudaStream_t, 0 = ok,
 * negative = error with a message from eqf_last_error().
 */
#ifndef EQF_B200_OPTIM_H_
#define EQF_B200_OPTIM_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EQF_OPTIM_THREADS 256   /* threads per CTA; each thread takes 4 elements per pass */
#define EQF_OPTIM_MAX_CTAS 1024 /* grid cap: past 4 * 256 * 1024 elements every CTA strides more than once */

const char* eqf_last_error(void);

/* partials: double[EQF_OPTIM_MAX_CTAS] scratch; norm, coef: one float each */
int eqf_flat_sqnorm(const float* g, int64_t n, float max_norm, double* partials, int32_t* tickets, float* norm,
                    float* coef, void* stream);

/* coef, lr: one float each; step: one int64, incremented by the call; ema may be NULL */
int eqf_flat_adamw(float* g, float* p, float* m, float* v, const float* decay, float* ema, int64_t n, const float* coef,
                   const float* lr, int64_t* step, double beta1, double beta2, float eps, double ema_decay,
                   int32_t* tickets, void* stream);

/* The argument checks of the two entry points on their own: host code only, nothing is launched or dereferenced.
 * Each entry point returns what its check returns before it launches anything. */
int eqf_flat_sqnorm_check(const float* g, int64_t n, float max_norm, const double* partials, const int32_t* tickets,
                          const float* norm, const float* coef);
int eqf_flat_adamw_check(const float* g, const float* p, const float* m, const float* v, const float* decay,
                         const float* ema, int64_t n, const float* coef, const float* lr, const int64_t* step,
                         double beta1, double beta2, const int32_t* tickets);

#ifdef __cplusplus
}
#endif
#endif
