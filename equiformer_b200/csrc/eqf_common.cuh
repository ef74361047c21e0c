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
constexpr int kMaxD = 7;                // degrees 0..3  (2l+1 <= 7)

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
int dtp_variant();                        // 0 scalar, 1 vec, 2 vec + TMA weights, 3 pipelined v3, 4 generated (env EQF_DTP_VARIANT)
int launch_forward_vec(const EqfPlan* plan, const EdgeArgs& a, bool tma, cudaStream_t stream);
int launch_grad_x_vec(const EqfPlan* plan, const EdgeArgs& a, bool with_w, cudaStream_t stream);
int launch_forward_v3(const EqfPlan* plan, const EdgeArgs& a, cudaStream_t stream);
int launch_backward_v3(const EqfPlan* plan, const EdgeArgs& a, bool with_w, cudaStream_t stream);
int backward_v3_grid(const EqfPlan* plan, long long E);

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
