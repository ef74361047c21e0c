// Gradient-norm clipping, AdamW and the model EMA on flat fp32 buffers: see include/eqf_b200_optim.h.
//
// Both kernels are one grid-stride pass over float4 slices (the tail of n % 4 elements goes to the first CTA) with a
// capped grid.  The step's scalars are read from device memory by thread 0 of each CTA, so a captured step replays with
// whatever the learning rate, the clip coefficient and the step count hold at replay time.  The CTA that finishes last
// (a completion ticket, the only atomic) finishes the call: eqf_flat_sqnorm sums the per-CTA partials in CTA order,
// eqf_flat_adamw writes the incremented step count once every CTA has read the old one.
//
// A scheduled step (eqf_flat_adamw_scheduled) runs the same kernel instances: the schedule descriptor travels in the
// kernel arguments, thread 0 of each CTA evaluates lr_at() from the step count instead of reading *lr, and the last CTA
// also writes the next step's rate.  lr_at() is __host__ __device__, so eqf_lr_at() hands the host the very function the
// kernel runs.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <string>

#include "eqf_b200_optim.h"

namespace eqf {

static thread_local std::string g_optim_error;
constexpr int kThreads = EQF_OPTIM_THREADS;
constexpr int kMaxCtas = EQF_OPTIM_MAX_CTAS;

static int fail(const char* msg) {
  g_optim_error = msg;
  return -1;
}

static int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return 0;
  g_optim_error = std::string(what) + ": " + cudaGetErrorString(e);
  return -2;
}

static bool aligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static unsigned grid_of(int64_t n) {
  const int64_t ctas = ((n >> 2) + kThreads - 1) / kThreads;
  return (unsigned)(ctas < 1 ? 1 : (ctas < kMaxCtas ? ctas : kMaxCtas));
}

// tree sum over the CTA in a fixed order; every thread gets the total
__device__ __forceinline__ double block_sum(double* red, double v) {
  red[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// thread 0: true in the CTA that finishes last (after every CTA's earlier writes are visible)
__device__ __forceinline__ bool last_cta(int32_t* tickets) {
  __threadfence();
  return atomicAdd(tickets, 1) == (int32_t)gridDim.x - 1;
}

__device__ __forceinline__ double sq4(float4 q) {
  return (double)q.x * q.x + (double)q.y * q.y + (double)q.z * q.z + (double)q.w * q.w;
}

__global__ void __launch_bounds__(kThreads) flat_sqnorm_kernel(const float* __restrict__ g, int64_t n, float max_norm,
                                                               double* part, int32_t* tickets, float* norm, float* coef) {
  __shared__ double red[kThreads];
  __shared__ bool last;
  const int64_t n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  double acc = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n4; i += (int64_t)gridDim.x * kThreads)
    acc += sq4(g4[i]);
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const double x = g[4 * n4 + threadIdx.x];
    acc += x * x;
  }
  acc = block_sum(red, acc);
  if (threadIdx.x == 0) {
    part[blockIdx.x] = acc;
    last = last_cta(tickets);
  }
  __syncthreads();
  if (!last) return;
  double tot = 0.0;
  for (int i = threadIdx.x; i < (int)gridDim.x; i += kThreads) tot += __ldcg(part + i);
  tot = block_sum(red, tot);
  if (threadIdx.x == 0) {
    const float nf = (float)sqrt(tot);
    const float c = max_norm / (nf + 1e-6f);
    *norm = nf;
    *coef = (c < 1.f || c != c) ? c : 1.f;      // torch.clamp(max=1) keeps a NaN
    *tickets = 0;
  }
}

struct AdamArgs {
  float* g;
  float* p;
  float* m;
  float* v;
  const float* decay;
  float* ema;
  int64_t n;
  const float* coef;
  float* lr;               // read by an unscheduled step, written by a scheduled one
  int64_t* step;
  double b1, b2;
  float eps, ema_w;
  int32_t* tickets;
  EqfLrSchedule sched;     // kind EQF_LR_NONE: the rate is *lr
};

// Products and sums rounded one by one: no fused multiply-add, so the device evaluates each schedule expression in the
// reference's operation order, as Python (and the host compiler, which contracts nothing on x86-64) does.
__host__ __device__ __forceinline__ double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}

__host__ __device__ __forceinline__ double add_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

// The rate of the step whose count before the step is t: include/eqf_b200_optim.h states each kind's expression, and
// the comments name the reference expression each line copies.
__host__ __device__ inline double lr_at(const EqfLrSchedule& s, int64_t t) {
  const double u = (double)(t / s.steps_per_unit);
  const double pi = 3.141592653589793;   // math.pi
  if (s.kind == EQF_LR_TIMM_COSINE) {
    // CosineLRScheduler._get_lr: warmup_lr_init + t * warmup_step, warmup_step = (base - warmup_lr_init) / warmup_t
    if (u < s.warmup) return add_rn(s.warmup_start, mul_rn(u, (s.base_lr - s.warmup_start) / s.warmup));
    // lr_min + 0.5 * (lr_max - lr_min) * (1 + math.cos(math.pi * t_curr / t_i)), first and only cycle
    if (u < s.total)
      return add_rn(s.min_value, mul_rn(mul_rn(0.5, s.base_lr - s.min_value), 1.0 + cos(mul_rn(pi, u) / s.total)));
    return s.min_value;
  }
  double lambda;
  if (u <= s.warmup) {
    // alpha = current_step / float(warmup_epochs); lr_warmup_factor * (1.0 - alpha) + alpha
    const double a = u / s.warmup;
    lambda = add_rn(mul_rn(s.warmup_start, 1.0 - a), a);
  } else if (s.kind == EQF_LR_OC20_MULTISTEP) {
    int idx = 0;                                           // bisect(lr_decay_epochs, current_step)
    for (int i = 0; i < s.n_milestones; ++i) idx += s.milestones[i] <= u;
    lambda = pow(s.gamma, (double)idx);                    // pow(lr_gamma, idx)
  } else if (u >= s.total) {
    lambda = s.min_value;
  } else {
    // lr_min_factor + 0.5 * (1 - lr_min_factor) * (1 + math.cos(math.pi * (current_step / max_epochs)))
    lambda = add_rn(s.min_value, mul_rn(mul_rn(0.5, 1.0 - s.min_value), 1.0 + cos(mul_rn(pi, u / s.total))));
  }
  return mul_rn(s.base_lr, lambda);                        // base_lr * lmbda(self.last_epoch)
}

struct AdamScalars {
  float coef, b1, one_m_b1, b2, one_m_b2, neg_lr, neg_step, sqrt_bc2, eps, ema_w;
  int64_t t;
};

// the operation order of FlatAdamW.step(): m, v, decoupled decay, then the bias-corrected update
__device__ __forceinline__ void adamw_one(const AdamScalars& s, float& g, float& p, float& m, float& v, float wd) {
  g *= s.coef;
  m = m * s.b1 + s.one_m_b1 * g;
  v = v * s.b2 + s.one_m_b2 * (g * g);
  p = p + s.neg_lr * (p * wd);
  const float denom = sqrtf(v) / s.sqrt_bc2 + s.eps;
  p = p + s.neg_step * (m / denom);
}

__device__ __forceinline__ void adamw4(const AdamScalars& s, float4& g, float4& p, float4& m, float4& v, float4 wd) {
  adamw_one(s, g.x, p.x, m.x, v.x, wd.x);
  adamw_one(s, g.y, p.y, m.y, v.y, wd.y);
  adamw_one(s, g.z, p.z, m.z, v.z, wd.z);
  adamw_one(s, g.w, p.w, m.w, v.w, wd.w);
}

__device__ __forceinline__ float lerp1(float e, float p, float w) { return e + w * (p - e); }

template <bool kEma>
__global__ void __launch_bounds__(kThreads) flat_adamw_kernel(AdamArgs a) {
  __shared__ AdamScalars sh;
  __shared__ bool last;
  if (threadIdx.x == 0) {
    const int64_t t = *a.step + 1;
    // a scheduled rate is rounded to float as a rate written by set_lr() is
    const double lr = a.sched.kind == EQF_LR_NONE ? (double)*a.lr : (double)(float)lr_at(a.sched, t - 1);
    sh.t = t;
    sh.coef = *a.coef;
    sh.b1 = (float)a.b1;
    sh.one_m_b1 = (float)(1.0 - a.b1);
    sh.b2 = (float)a.b2;
    sh.one_m_b2 = (float)(1.0 - a.b2);
    sh.neg_lr = (float)-lr;
    sh.neg_step = (float)(-lr / (1.0 - pow(a.b1, (double)t)));
    sh.sqrt_bc2 = (float)sqrt(1.0 - pow(a.b2, (double)t));
    sh.eps = a.eps;
    sh.ema_w = a.ema_w;
  }
  __syncthreads();
  const AdamScalars s = sh;
  const bool store_g = s.coef != 1.f;        // g * 1 == g: an unclipped step leaves the gradient as it is
  const int64_t n4 = a.n >> 2;
  float4* g4 = reinterpret_cast<float4*>(a.g);
  float4* p4 = reinterpret_cast<float4*>(a.p);
  float4* m4 = reinterpret_cast<float4*>(a.m);
  float4* v4 = reinterpret_cast<float4*>(a.v);
  const float4* d4 = reinterpret_cast<const float4*>(a.decay);
  float4* e4 = reinterpret_cast<float4*>(a.ema);
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n4; i += (int64_t)gridDim.x * kThreads) {
    float4 g = g4[i], p = p4[i], m = m4[i], v = v4[i];
    adamw4(s, g, p, m, v, d4[i]);
    if (store_g) g4[i] = g;
    p4[i] = p;
    m4[i] = m;
    v4[i] = v;
    if (kEma) {
      float4 e = e4[i];
      e.x = lerp1(e.x, p.x, s.ema_w);
      e.y = lerp1(e.y, p.y, s.ema_w);
      e.z = lerp1(e.z, p.z, s.ema_w);
      e.w = lerp1(e.w, p.w, s.ema_w);
      e4[i] = e;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (a.n & 3)) {
    const int64_t i = 4 * n4 + threadIdx.x;
    float g = a.g[i], p = a.p[i], m = a.m[i], v = a.v[i];
    adamw_one(s, g, p, m, v, a.decay[i]);
    a.g[i] = g;
    a.p[i] = p;
    a.m[i] = m;
    a.v[i] = v;
    if (kEma) a.ema[i] = lerp1(a.ema[i], p, s.ema_w);
  }
  __syncthreads();
  if (threadIdx.x == 0) last = last_cta(a.tickets);
  __syncthreads();
  if (last && threadIdx.x == 0) {
    *a.step = s.t;
    if (a.sched.kind != EQF_LR_NONE) *a.lr = (float)lr_at(a.sched, s.t);   // no CTA reads *lr in a scheduled step
    *a.tickets = 0;
  }
}

}  // namespace eqf

using namespace eqf;

extern "C" const char* eqf_last_error(void) { return g_optim_error.c_str(); }

extern "C" int eqf_flat_sqnorm_check(const float* g, int64_t n, float max_norm, const double* partials,
                                     const int32_t* tickets, const float* norm, const float* coef) {
  if (n <= 0) return fail("eqf_flat_sqnorm: n must be positive");
  if (!g || !partials || !tickets || !norm || !coef) return fail("eqf_flat_sqnorm: null pointer");
  if (!aligned(g)) return fail("eqf_flat_sqnorm: the gradient buffer must be 16-byte aligned");
  if (!(max_norm > 0.f)) return fail("eqf_flat_sqnorm: max_norm must be positive");
  return 0;
}

extern "C" int eqf_flat_sqnorm(const float* g, int64_t n, float max_norm, double* partials, int32_t* tickets, float* norm,
                               float* coef, void* stream) {
  const int rc = eqf_flat_sqnorm_check(g, n, max_norm, partials, tickets, norm, coef);
  if (rc) return rc;
  flat_sqnorm_kernel<<<grid_of(n), kThreads, 0, (cudaStream_t)stream>>>(g, n, max_norm, partials, tickets, norm, coef);
  return check_launch("flat_sqnorm_kernel launch");
}

static int launch_adamw(const AdamArgs& a, void* stream) {
  if (a.ema)
    flat_adamw_kernel<true><<<grid_of(a.n), kThreads, 0, (cudaStream_t)stream>>>(a);
  else
    flat_adamw_kernel<false><<<grid_of(a.n), kThreads, 0, (cudaStream_t)stream>>>(a);
  return check_launch("flat_adamw_kernel launch");
}

extern "C" int eqf_flat_adamw_check(const float* g, const float* p, const float* m, const float* v, const float* decay,
                                    const float* ema, int64_t n, const float* coef, const float* lr, const int64_t* step,
                                    double beta1, double beta2, const int32_t* tickets) {
  if (n <= 0) return fail("eqf_flat_adamw: n must be positive");
  if (!g || !p || !m || !v || !decay || !coef || !lr || !step || !tickets) return fail("eqf_flat_adamw: null pointer");
  if (!aligned(g) || !aligned(p) || !aligned(m) || !aligned(v) || !aligned(decay) || (ema && !aligned(ema)))
    return fail("eqf_flat_adamw: every buffer must be 16-byte aligned");
  if (!(beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0)) return fail("eqf_flat_adamw: betas must be in [0, 1)");
  return 0;
}

extern "C" int eqf_flat_adamw(float* g, float* p, float* m, float* v, const float* decay, float* ema, int64_t n,
                              const float* coef, const float* lr, int64_t* step, double beta1, double beta2, float eps,
                              double ema_decay, int32_t* tickets, void* stream) {
  const int rc = eqf_flat_adamw_check(g, p, m, v, decay, ema, n, coef, lr, step, beta1, beta2, tickets);
  if (rc) return rc;
  AdamArgs a{g, p, m, v, decay, ema, n, coef, const_cast<float*>(lr), step, beta1, beta2, eps,
             (float)(1.0 - ema_decay), tickets, EqfLrSchedule{}};
  return launch_adamw(a, stream);
}

extern "C" int eqf_lr_schedule_check(const EqfLrSchedule* s) {
  if (!s) return fail("eqf_lr_schedule: null descriptor");
  const bool timm = s->kind == EQF_LR_TIMM_COSINE, multistep = s->kind == EQF_LR_OC20_MULTISTEP;
  if (s->kind != EQF_LR_OC20_COSINE && !multistep && !timm) return fail("eqf_lr_schedule: unknown kind");
  if (!std::isfinite(s->warmup) || (timm ? s->warmup < 0.0 : s->warmup <= 0.0))
    return fail(timm ? "eqf_lr_schedule: the warm-up length must be finite and >= 0"
                     : "eqf_lr_schedule: the warm-up length must be finite and positive (the warm-up divides by it)");
  if (!multistep && !(std::isfinite(s->total) && s->total > 0.0))
    return fail("eqf_lr_schedule: the total length must be finite and positive");
  if (s->steps_per_unit < 1) return fail("eqf_lr_schedule: steps_per_unit must be at least 1");
  if (s->n_milestones < 0 || s->n_milestones > EQF_LR_MAX_MILESTONES)
    return fail("eqf_lr_schedule: at most EQF_LR_MAX_MILESTONES milestones");
  for (int i = 0; i < s->n_milestones; ++i) {
    if (!std::isfinite(s->milestones[i])) return fail("eqf_lr_schedule: milestones must be finite");
    if (i && s->milestones[i] < s->milestones[i - 1]) return fail("eqf_lr_schedule: milestones must be sorted");
  }
  // every rate is base_lr times a value between the warm-up start, 1, the floor and gamma^k (OC20), or lies between
  // warmup_start, base_lr and min_value (timm): non-negative finite parameters and a finite largest product suffice
  const double pars[] = {s->base_lr, s->warmup_start, s->min_value, multistep ? s->gamma : 0.0};
  for (double x : pars)
    if (!(std::isfinite(x) && x >= 0.0)) return fail("eqf_lr_schedule: a parameter gives a negative or non-finite rate");
  if (!timm) {
    double top = s->warmup_start > 1.0 ? s->warmup_start : 1.0;
    if (s->min_value > top) top = s->min_value;
    if (multistep && s->gamma > 1.0) top = pow(s->gamma, (double)s->n_milestones);
    if (!std::isfinite(s->base_lr * top)) return fail("eqf_lr_schedule: a parameter gives a negative or non-finite rate");
  }
  return 0;
}

extern "C" int eqf_lr_at(const EqfLrSchedule* s, int64_t t, double* out) {
  const int rc = eqf_lr_schedule_check(s);
  if (rc) return rc;
  if (t < 0 || !out) return fail("eqf_lr_at: the step count must be >= 0 and out given");
  *out = lr_at(*s, t);
  return 0;
}

extern "C" int eqf_flat_adamw_scheduled(float* g, float* p, float* m, float* v, const float* decay, float* ema, int64_t n,
                                        const float* coef, float* lr, int64_t* step, double beta1, double beta2,
                                        float eps, double ema_decay, int32_t* tickets, const EqfLrSchedule* schedule,
                                        void* stream) {
  int rc = eqf_flat_adamw_check(g, p, m, v, decay, ema, n, coef, lr, step, beta1, beta2, tickets);
  if (!rc) rc = eqf_lr_schedule_check(schedule);
  if (rc) return rc;
  AdamArgs a{g, p, m, v, decay, ema, n, coef, lr, step, beta1, beta2, eps, (float)(1.0 - ema_decay), tickets, *schedule};
  return launch_adamw(a, stream);
}
