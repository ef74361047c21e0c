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

/* Learning-rate schedules of the reference trainers, evaluated from the optimiser step count t (the count BEFORE the
 * step: the k-th step, k = 0, 1, ..., runs at lr(t = k)).  The unit u is t / steps_per_unit (integer division):
 * 1 for schedules stepped every iteration (OC20), the iterations per epoch for timm's per-epoch schedules.
 *
 *   EQF_LR_OC20_COSINE     oc20/trainer/lr_scheduler.py CosineLRLambda under torch's LambdaLR, lr = base_lr * lambda(u):
 *                          u <= W: a = u / W, lambda = f (1 - a) + a;  u >= T: lambda = m;
 *                          else lambda = m + 0.5 (1 - m) (1 + cos(pi (u / T)))
 *   EQF_LR_OC20_MULTISTEP  MultistepLRLambda: the same warm-up, then lambda = gamma ^ bisect_right(milestones, u)
 *   EQF_LR_TIMM_COSINE     timm 0.4.12 CosineLRScheduler._get_lr as create_scheduler builds it (t_mul 1, cycle_limit 1, no
 *                          noise, warmup_prefix False), restated here, never executed against timm:
 *                          u < W: f + u ((base_lr - f) / W);  u < T: m + 0.5 (base_lr - m) (1 + cos((pi u) / T));
 *                          else m
 *
 * W = warmup, f = warmup_start (a factor for OC20, a rate for timm), T = total, m = min_value (a factor for OC20, a rate
 * for timm).  Every expression is evaluated in double, in the order written above. */
#define EQF_LR_MAX_MILESTONES 8

enum { EQF_LR_NONE = 0, EQF_LR_OC20_COSINE = 1, EQF_LR_OC20_MULTISTEP = 2, EQF_LR_TIMM_COSINE = 3 };

typedef struct EqfLrSchedule {
  int32_t kind;           /* EQF_LR_* */
  int32_t n_milestones;   /* EQF_LR_OC20_MULTISTEP: milestones used, at most EQF_LR_MAX_MILESTONES */
  int64_t steps_per_unit; /* >= 1 */
  double base_lr;
  double warmup;          /* W, in units */
  double warmup_start;
  double total;           /* T, in units (unused by EQF_LR_OC20_MULTISTEP) */
  double min_value;       /* the floor: a factor for OC20 (lr_min_factor), a rate for timm (min_lr) */
  double gamma;           /* EQF_LR_OC20_MULTISTEP */
  double milestones[EQF_LR_MAX_MILESTONES]; /* ascending, in units */
} EqfLrSchedule;

/* 0 when `s` describes a schedule the kernel can run; refused: an unknown kind, W <= 0 (W < 0 for timm, whose warm-up
 * may be empty), T <= 0 for the cosine kinds, steps_per_unit < 1, more than EQF_LR_MAX_MILESTONES milestones or
 * milestones out of order, and any parameter that can make a rate negative or non-finite.  Host code only. */
int eqf_lr_schedule_check(const EqfLrSchedule* s);
/* *out = the rate of the step whose count before the step is t (t >= 0), by the function the kernel runs.  Host code. */
int eqf_lr_at(const EqfLrSchedule* s, int64_t t, double* out);

/* eqf_flat_adamw with the learning rate taken from `schedule` (checked before launch): thread 0 of every CTA evaluates
 * lr(step) instead of reading *lr, and the call leaves (float) lr(step + 1), the next step's rate, in *lr next to the
 * incremented step count.  Nothing is read from the host, so a captured step replays a whole schedule. */
int eqf_flat_adamw_scheduled(float* g, float* p, float* m, float* v, const float* decay, float* ema, int64_t n,
                             const float* coef, float* lr, int64_t* step, double beta1, double beta2, float eps,
                             double ema_decay, int32_t* tickets, const EqfLrSchedule* schedule, void* stream);

#ifdef __cplusplus
}
#endif
#endif
