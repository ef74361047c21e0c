// Metric terms of an evaluation pass, added to a float64 accumulator on the device: see include/eqf_b200_eval.h.
//
// The graph- and atom-level kernels are one grid-stride pass over the rows with a capped grid.  Each thread sums its
// rows' terms in double; the CTA reduces them in a fixed tree and writes one partial per term.  The CTA that finishes
// last (a completion ticket, the only atomic) sums the partials in CTA order and adds them and the row count to the
// accumulator, as eqf_flat_sqnorm does, so a repeated pass is bitwise equal.  The terms are formed with the _rn
// intrinsics: no multiply-add is contracted, so each is rounded as the reference's float32 tensor expression rounds it.
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "eqf_b200_eval.h"

namespace eqf {

static thread_local std::string g_eval_error;
constexpr int kThreads = EQF_EVAL_THREADS;
constexpr int kMaxCtas = EQF_EVAL_MAX_CTAS;
static_assert(EQF_EVAL_SCRATCH == EQF_EVAL_MAX_CTAS * EQF_EVAL_MAX_TERMS, "partials scratch");

static int fail(const char* msg) {
  g_eval_error = msg;
  return -1;
}

static int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return 0;
  g_eval_error = std::string(what) + ": " + cudaGetErrorString(e);
  return -2;
}

static unsigned grid_of(int64_t rows) {
  const int64_t ctas = (rows + kThreads - 1) / kThreads;
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

// Reduce the K per-thread sums of the CTA to its partials; the CTA that finishes last adds the CTA-ordered totals to
// acc[0..K-1] and `count` to acc[K], and resets the ticket.
template <int K>
__device__ __forceinline__ void finish(double (&v)[K], double count, double* part, int32_t* tickets, double* acc) {
  __shared__ double red[kThreads];
  __shared__ bool last;
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = block_sum(red, v[k]);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) part[blockIdx.x * K + k] = v[k];
    __threadfence();
    last = atomicAdd(tickets, 1) == (int32_t)gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double tot = 0.0;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += kThreads) tot += __ldcg(part + i * K + k);
    tot = block_sum(red, tot);
    if (threadIdx.x == 0) acc[k] += tot;
  }
  if (threadIdx.x == 0) {
    acc[K] += count;
    *tickets = 0;
  }
}

__global__ void __launch_bounds__(kThreads) eval_graph_kernel(const float* __restrict__ pred, const float* __restrict__ y,
                                                              int64_t n, float mean, float std, float thr, double* part,
                                                              int32_t* tickets, double* acc) {
  double v[4] = {0.0, 0.0, 0.0, 0.0};
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const float p = pred[i], t = y[i];
    const float e = __fsub_rn(__fadd_rn(__fmul_rn(p, std), mean), t);      // pred * std + mean - y
    const float ae = fabsf(e);
    v[0] += (double)ae;
    v[1] += (double)__fmul_rn(e, e);
    v[2] += ae < thr ? 1.0 : 0.0;                                          // false for NaN
    v[3] += (double)fabsf(__fsub_rn(p, __fdiv_rn(__fsub_rn(t, mean), std)));   // pred - (y - mean) / std
  }
  finish<4>(v, (double)n, part, tickets, acc);
}

__global__ void __launch_bounds__(kThreads) eval_atom_kernel(const float* __restrict__ pred, const float* __restrict__ dy,
                                                             int64_t rows, const int64_t* n_atoms, float std,
                                                             double* part, int32_t* tickets, double* acc) {
  int64_t n = *n_atoms;
  n = n < 0 ? 0 : (n < rows ? n : rows);
  double v[2] = {0.0, 0.0};
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    float q2 = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float p = pred[3 * i + c], t = dy[3 * i + c];
      v[0] += (double)fabsf(__fsub_rn(__fmul_rn(p, std), t));              // pred_dy * std - dy
      const float q = __fsub_rn(p, __fdiv_rn(t, std));                     // pred_dy - dy / std
      q2 = c == 0 ? __fmul_rn(q, q) : __fadd_rn(q2, __fmul_rn(q, q));
    }
    v[1] += (double)sqrtf(q2);
  }
  finish<2>(v, (double)n, part, tickets, acc);
}

__global__ void eval_batch_kernel(const float* loss, double* acc) {
  if (threadIdx.x == 0) {
    if (loss) acc[0] += (double)*loss;
    acc[1] += 1.0;
  }
}

}  // namespace eqf

using namespace eqf;

extern "C" const char* eqf_last_error(void) { return g_eval_error.c_str(); }

extern "C" int eqf_eval_graph_check(const float* pred, const float* y, int64_t n_graphs, const double* partials,
                                    const int32_t* tickets, const double* acc) {
  if (n_graphs <= 0) return fail("eqf_eval_graph: n_graphs must be positive");
  if (!pred || !y || !partials || !tickets || !acc) return fail("eqf_eval_graph: null pointer");
  return 0;
}

extern "C" int eqf_eval_graph(const float* pred, const float* y, int64_t n_graphs, float mean, float std, float threshold,
                              double* partials, int32_t* tickets, double* acc, void* stream) {
  const int rc = eqf_eval_graph_check(pred, y, n_graphs, partials, tickets, acc);
  if (rc) return rc;
  eval_graph_kernel<<<grid_of(n_graphs), kThreads, 0, (cudaStream_t)stream>>>(pred, y, n_graphs, mean, std, threshold,
                                                                              partials, tickets, acc);
  return check_launch("eval_graph_kernel launch");
}

extern "C" int eqf_eval_atom_check(const float* pred_dy, const float* dy, int64_t n_rows, const int64_t* n_atoms,
                                   const double* partials, const int32_t* tickets, const double* acc) {
  if (n_rows <= 0) return fail("eqf_eval_atom: n_rows must be positive");
  if (!pred_dy || !dy || !n_atoms || !partials || !tickets || !acc) return fail("eqf_eval_atom: null pointer");
  return 0;
}

extern "C" int eqf_eval_atom(const float* pred_dy, const float* dy, int64_t n_rows, const int64_t* n_atoms, float std,
                             double* partials, int32_t* tickets, double* acc, void* stream) {
  const int rc = eqf_eval_atom_check(pred_dy, dy, n_rows, n_atoms, partials, tickets, acc);
  if (rc) return rc;
  eval_atom_kernel<<<grid_of(n_rows), kThreads, 0, (cudaStream_t)stream>>>(pred_dy, dy, n_rows, n_atoms, std, partials,
                                                                           tickets, acc);
  return check_launch("eval_atom_kernel launch");
}

extern "C" int eqf_eval_batch_check(const float* loss, const double* acc) {
  (void)loss;
  if (!acc) return fail("eqf_eval_batch: null pointer");
  return 0;
}

extern "C" int eqf_eval_batch(const float* loss, double* acc, void* stream) {
  const int rc = eqf_eval_batch_check(loss, acc);
  if (rc) return rc;
  eval_batch_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(loss, acc);
  return check_launch("eval_batch_kernel launch");
}
