// De-normalised OC20 IS2RE predictions of one batch: see include/eqf_b200_predict.h.
//
// One grid-stride pass over max(n_graphs, n_rows) rows with a capped grid; a thread writes row i's energy when
// i < n_graphs and its three position components when i < n_rows.  The arithmetic is the _rn intrinsics, so no
// multiply-add is contracted and each operation rounds as the reference's eager float32 tensor expression does.
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "eqf_b200_predict.h"

namespace eqf {

static thread_local std::string g_predict_error;
constexpr int kThreads = EQF_PREDICT_THREADS;
constexpr int kMaxCtas = EQF_PREDICT_MAX_CTAS;

static int fail(const char* msg) {
  g_predict_error = msg;
  return -1;
}

__global__ void __launch_bounds__(kThreads) predict_is2re_kernel(const float* __restrict__ energy, int64_t n_graphs,
                                                                 float mean, float std, const float* __restrict__ pos,
                                                                 const float* __restrict__ delta,
                                                                 const int64_t* __restrict__ tags, int64_t n_rows,
                                                                 float pos_std, float* __restrict__ energy_out,
                                                                 float* __restrict__ pos_out) {
  const int64_t rows = n_graphs > n_rows ? n_graphs : n_rows;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < rows; i += (int64_t)gridDim.x * kThreads) {
    if (i < n_graphs) energy_out[i] = __fadd_rn(__fmul_rn(energy[i], std), mean);        // energy * std + mean
    if (i < n_rows) {
      const bool moves = tags[i] > 0;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float p = pos[3 * i + c];
        // pos + (delta * pos_std + 0): the positions normaliser's denorm (mean 0), then the masked add
        pos_out[3 * i + c] = moves ? __fadd_rn(p, __fadd_rn(__fmul_rn(delta[3 * i + c], pos_std), 0.0f)) : p;
      }
    }
  }
}

}  // namespace eqf

using namespace eqf;

extern "C" const char* eqf_last_error(void) { return g_predict_error.c_str(); }

extern "C" int eqf_predict_is2re_check(const float* energy, int64_t n_graphs, const float* pos, const float* delta,
                                       const int64_t* tags, int64_t n_rows, const float* energy_out,
                                       const float* pos_out) {
  if (n_graphs < 0) return fail("eqf_predict_is2re: n_graphs must not be negative");
  if (n_rows < 0) return fail("eqf_predict_is2re: n_rows must not be negative");
  if (!energy || !energy_out) return fail("eqf_predict_is2re: null pointer (energy, energy_out)");
  const int given = (pos != nullptr) + (delta != nullptr) + (tags != nullptr) + (pos_out != nullptr);
  if (given != 0 && given != 4)
    return fail("eqf_predict_is2re: null pointer: pos, delta, tags and pos_out are all given or all NULL");
  return 0;
}

extern "C" int eqf_predict_is2re(const float* energy, int64_t n_graphs, float mean, float std, const float* pos,
                                 const float* delta, const int64_t* tags, int64_t n_rows, float pos_std,
                                 float* energy_out, float* pos_out, void* stream) {
  const int rc = eqf_predict_is2re_check(energy, n_graphs, pos, delta, tags, n_rows, energy_out, pos_out);
  if (rc) return rc;
  if (!delta) n_rows = 0;
  const int64_t rows = n_graphs > n_rows ? n_graphs : n_rows;
  if (rows == 0) return 0;
  const int64_t ctas = (rows + kThreads - 1) / kThreads;
  predict_is2re_kernel<<<(unsigned)(ctas < kMaxCtas ? ctas : kMaxCtas), kThreads, 0, (cudaStream_t)stream>>>(
      energy, n_graphs, mean, std, pos, delta, tags, n_rows, pos_std, energy_out, pos_out);
  const cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return 0;
  g_predict_error = std::string("predict_is2re_kernel launch: ") + cudaGetErrorString(e);
  return -2;
}
