// eqf_common.cuh - shared device/host definitions for libeqf_b200.so (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>

#include "../../include/eqf_b200.h"

struct EqfPlan;

namespace eqf {

constexpr int kThreads = 256;           // threads per CTA for the edge kernels
constexpr int kWarps = kThreads / 32;
constexpr int kMaxD = 7;                // degrees 0..3  (2l+1 <= 7): fused DTP -> linear kernel (eqf_fused.cu)
// Largest in1 / output degree of a depth-wise plan.  libeqf_b200.so keeps 3; the table-walk DTP sources (eqf_abi.cu,
// eqf_dtp.cu, eqf_dtp_vec.cu) are built a second time with -DEQF_MAX_DEGREE=4 into libeqf_b200_l4.so, so the degree-4
// branches never enter the kernels (and the register allocation) of the l <= 3 library.
#ifndef EQF_MAX_DEGREE
#define EQF_MAX_DEGREE 3
#endif
constexpr int kMaxDtpD = 2 * EQF_MAX_DEGREE + 1;
#if EQF_MAX_DEGREE >= 4
#define EQF_CASE_D9(NAME, ...) case 9: { constexpr int NAME = 9; __VA_ARGS__; } break;
#else
#define EQF_CASE_D9(NAME, ...)
#endif

// Device-side path record (one Clebsch-Gordan path); mirrors EqfPathDesc + derived fields.
struct PathDev {
  int d1, d2, d3;   // 2l+1 of in1, in2, out
  int mul;          // channels
  int xb;           // in1 block
  int y_off;        // offset of the l2 SH in an edge_attr row
  int og;           // output group
  int koff;         // channel offset inside the output group
  int w_off;        // offset in the weight row
  int cg_off;       // offset in the dense CG table [d1][d2][d3]
  int m_off;        // offset in the per-edge M scratch [d1][d3]
  int pad;
};
static_assert(sizeof(PathDev) == 48, "PathDev layout");

// One path's per-edge coupling matrix M_p[i, k] (i < D1, k < D3) as the table-walk DTP kernels read it.  Up to 7 x 7 it is
// copied to registers once per task.  A degree-4 side would make that up to 9 x 9 = 81 registers, and since a kernel's
// register count is the maximum over all of its branches, it would raise the count (or spill) for every l <= 3 plan too;
// so a path with a degree-4 input or output reads each entry from shared memory where it is used (a broadcast load), and
// its task loops over the output components k one at a time (`#pragma unroll 1`), so that neither the tile nor a row of
// cotangents is ever live in registers at once.
template <int D1, int D3, bool IN_REGS = (D1 <= 7 && D3 <= 7)>
struct MTile {
  static constexpr bool kInRegs = true;
  float v[D1][D3];
  __device__ __forceinline__ explicit MTile(const float* __restrict__ Mp) {
#pragma unroll
    for (int i = 0; i < D1; ++i)
#pragma unroll
      for (int k = 0; k < D3; ++k) v[i][k] = Mp[i * D3 + k];
  }
  __device__ __forceinline__ float operator()(int i, int k) const { return v[i][k]; }
};
template <int D1, int D3>
struct MTile<D1, D3, false> {
  static constexpr bool kInRegs = false;
  const float* __restrict__ p;
  __device__ __forceinline__ explicit MTile(const float* __restrict__ Mp) : p(Mp) {}
  __device__ __forceinline__ float operator()(int i, int k) const { return p[i * D3 + k]; }
};

// Header passed by value to every edge kernel; offsets index the int/float blob in global memory.
struct PlanHdr {
  int n_paths, n_in1, n_out, d_y, w_numel, m_size, cg_len;
  int n_wtasks;     // (path, 32-channel chunk) tasks per edge   [forward / grad_w / grad_y]
  int n_xtasks;     // (in1 block, 32-channel chunk) tasks per edge [grad_x / grad_xw]
  int blob_words;
  int off_paths, off_cg, off_mdesc, off_wtasks, off_xtasks, off_xbstart, off_xbpaths;
  int te;           // edges per tile
  // vectorised kernels (eqf_dtp_vec.cu): per-tile task tables, lanes per edge / edges per warp of each in1 block
  int vec_ok, n_vwtasks, n_vxtasks, off_vwtasks, off_vxtasks;
  int in1_lpe[EQF_MAX_BLOCKS], in1_epw[EQF_MAX_BLOCKS];
  int in1_lpe_shift[EQF_MAX_BLOCKS];   // log2(lanes per edge) or -1 when not a power of two
  int in1_off[EQF_MAX_BLOCKS];         // float offset of each in1 block inside one [d_in] row
  int d_in;                            // floats per in1 row (all blocks)
  int in1_d[EQF_MAX_BLOCKS], in1_mul[EQF_MAX_BLOCKS];
  int out_d[EQF_MAX_BLOCKS], out_mul[EQF_MAX_BLOCKS];
};

struct EdgeArgs {
  const float* x[EQF_MAX_BLOCKS];
  const float* x2[EQF_MAX_BLOCKS];
  const long long* src;
  const long long* dst;
  const float* y;
  const float* w;
  const float* w_off;            // optional [W] offset added to every row of w (radial offset, fused into the load)
  int w_shared;
  const float* g[EQF_MAX_BLOCKS];
  float* out[EQF_MAX_BLOCKS];   // forward outputs (per output group)
  float* gx[EQF_MAX_BLOCKS];    // grad_x outputs (per in1 block)
  float* gw;                    // [E][W] or [grid][W]
  float* gy;                    // [E][d_y]
  long long E;
};

void set_error(const std::string& msg);
int check_cuda(cudaError_t err, const char* what);
int ensure_device(const EqfPlan* plan);  // uploads the table blob on first use
// plan-specialised kernels emitted by equiformer_b200/codegen.py (csrc/gen/*.cu), matched by plan hash
struct GeneratedKernels {
  unsigned long long signature;
  const char* tag;
  int (*forward)(const EqfPlan*, const EdgeArgs&, cudaStream_t);
  int (*backward)(const EqfPlan*, const EdgeArgs&, bool with_w, cudaStream_t);
  int (*grad_y)(const EqfPlan*, const EdgeArgs&, cudaStream_t);
  int (*partial_rows)(const EqfPlan*, long long);
};
int register_generated(const GeneratedKernels* k);
const GeneratedKernels* find_generated(unsigned long long signature);
int launch_forward_vec(const EqfPlan* plan, const EdgeArgs& a, bool tma, cudaStream_t stream);
int launch_grad_x_vec(const EqfPlan* plan, const EdgeArgs& a, bool with_w, cudaStream_t stream);

}  // namespace eqf

struct EqfPlan {
  eqf::PlanHdr hdr;
  std::vector<uint32_t> blob;   // host copy
  uint32_t* d_blob = nullptr;   // device copy
  int device = -1;
  int sm_count = 132;
  size_t smem_bytes = 0;        // dynamic shared memory per CTA (scalar kernels)
  size_t smem_bytes_vec_fwd = 0;  // vector forward (includes the TMA weight ring)
  size_t smem_bytes_vec_bwd = 0;  // vector grad_x / grad_xw
  unsigned long long signature = 0;            // FNV-1a of the path table (codegen.plan_signature)
  const eqf::GeneratedKernels* gen = nullptr;  // plan-specialised kernels when the signature is known
};
