// eqf_dtp.cu - the depth-wise tensor product (DTP) contraction family for sm_90a.
//
// Reference work replaced: o3.TensorProduct('uvu') inside TensorProductRescale
// (nets/tensor_product_rescale.py:33-37,126) as instantiated by DepthwiseTensorProduct
// (nets/graph_attention_transformer.py:157-183): ~4 eager launches per CG path + cat, and the
// autograd graph e3nn derives from it.  Here the quadrilinear form
//     S(x, y, w, g) = sum_e sum_p sum_u w[e,p,u] sum_ijk C_p[i,j,k] x[e,i,u] y[e,j] g[e,k,koff_p+u]
// is differentiated by hand: four kernels produce dS/dg (forward), dS/dx, dS/dw, dS/dy; the family is
// closed under differentiation, so first and second derivatives reuse the same kernels.
//
// Data layout (HBM): planar irrep blocks [E][2l+1][mul] - lanes run over channels u, so every global
// access of a warp is one contiguous 128-byte line.  Per edge the kernel first folds the edge
// harmonics into small matrices M_p[i,k] = sum_j C_p[i,j,k] y[e,j] (shared memory), after which each
// path is a (2l1+1)x(2l3+1) mat-vec per channel held entirely in registers.
//
// HBM-bound streaming kernels: per edge the forward moves 4*(D_in + D_y + W + D_out) bytes for about
// 2*sum_p mul*(2l1+1)*(2l3+1) flops (QM9 Lmax=2: 18 340 B vs 17 kflop).
#include <mutex>
#include <unordered_map>

#include "eqf_common.cuh"

namespace eqf {

// ------------------------------------------------------------------------------------------------
// shared-memory carve-up
struct Smem {
  const PathDev* paths;
  const float* cg;
  const int* mdesc;
  const int2* wtasks;
  const int2* xtasks;
  const int* xbstart;
  const int* xbpaths;
  float* M;      // [te][m_size]
  float* ysh;    // [te][d_y]
  float* extra;  // kernel specific
};

__device__ __forceinline__ Smem carve(const PlanHdr& h, const uint32_t* __restrict__ blob, uint32_t* smem) {
  for (int i = threadIdx.x; i < h.blob_words; i += blockDim.x) smem[i] = blob[i];
  Smem s;
  s.paths = reinterpret_cast<const PathDev*>(smem + h.off_paths);
  s.cg = reinterpret_cast<const float*>(smem + h.off_cg);
  s.mdesc = reinterpret_cast<const int*>(smem + h.off_mdesc);
  s.wtasks = reinterpret_cast<const int2*>(smem + h.off_wtasks);
  s.xtasks = reinterpret_cast<const int2*>(smem + h.off_xtasks);
  s.xbstart = reinterpret_cast<const int*>(smem + h.off_xbstart);
  s.xbpaths = reinterpret_cast<const int*>(smem + h.off_xbpaths);
  float* f = reinterpret_cast<float*>(smem + h.blob_words);
  s.M = f;
  s.ysh = s.M + h.te * h.m_size;
  s.extra = s.ysh + h.te * h.d_y;
  return s;
}

// Load the y tile and fold it into the per-edge matrices M_p[i,k]; ends with __syncthreads().
__device__ __forceinline__ void stage_tile(const PlanHdr& h, const Smem& s, const float* __restrict__ y,
                                           long long e0, long long E) {
  const int ny = h.te * h.d_y;
  for (int i = threadIdx.x; i < ny; i += blockDim.x) {
    long long gi = e0 * h.d_y + i;
    s.ysh[i] = (gi < E * h.d_y) ? __ldg(y + gi) : 0.f;
  }
  __syncthreads();
  const int nm = h.te * h.m_size;
  for (int idx = threadIdx.x; idx < nm; idx += blockDim.x) {
    const int te = idx / h.m_size;
    const int m = idx - te * h.m_size;
    const int desc = s.mdesc[m];
    const PathDev& P = s.paths[desc >> 8];
    const int i = (desc >> 4) & 15, k = desc & 15;
    const float* c = s.cg + P.cg_off + i * P.d2 * P.d3 + k;
    const float* yy = s.ysh + te * h.d_y + P.y_off;
    float acc = 0.f;
    for (int j = 0; j < P.d2; ++j) acc = fmaf(c[j * P.d3], yy[j], acc);
    s.M[idx] = acc;
  }
  __syncthreads();
}

#define EQF_DISPATCH_D(val, NAME, ...)                       \
  switch (val) {                                             \
    case 1: { constexpr int NAME = 1; __VA_ARGS__; } break;  \
    case 3: { constexpr int NAME = 3; __VA_ARGS__; } break;  \
    case 5: { constexpr int NAME = 5; __VA_ARGS__; } break;  \
    case 7: { constexpr int NAME = 7; __VA_ARGS__; } break;  \
    default: break;                                          \
  }

template <int D1>
__device__ __forceinline__ void load_x(const EdgeArgs& a, int xb, int mul, long long e, int u, float (&xi)[D1]) {
  const long long rs = a.src ? a.src[e] : e;
  const float* p = a.x[xb] + (rs * D1) * mul + u;
#pragma unroll
  for (int i = 0; i < D1; ++i) xi[i] = __ldg(p + (long long)i * mul);
  if (a.x2[xb] != nullptr) {
    const long long rd = a.dst[e];
    const float* q = a.x2[xb] + (rd * D1) * mul + u;
#pragma unroll
    for (int i = 0; i < D1; ++i) xi[i] += __ldg(q + (long long)i * mul);
  }
}

template <int D1, int D3>
__device__ __forceinline__ void load_M(const float* __restrict__ Mp, float (&M)[D1][D3]) {
#pragma unroll
  for (int i = 0; i < D1; ++i)
#pragma unroll
    for (int k = 0; k < D3; ++k) M[i][k] = Mp[i * D3 + k];
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------
// forward: out[og][e,k,koff+u] = w * sum_i x_i M[i,k]
template <int D1, int D3>
__device__ __forceinline__ void fwd_task(const PlanHdr& h, const EdgeArgs& a, const PathDev& P, const float* Mp,
                                         long long e, int u) {
  float M[D1][D3];
  load_M<D1, D3>(Mp, M);
  if (u >= P.mul) return;
  float xi[D1];
  load_x<D1>(a, P.xb, P.mul, e, u, xi);
  const float wv = __ldg(a.w + (a.w_shared ? 0 : e * h.w_numel) + P.w_off + u);
  const int K = h.out_mul[P.og];
  float* o = a.out[P.og] + (e * D3) * K + P.koff + u;
#pragma unroll
  for (int k = 0; k < D3; ++k) {
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < D1; ++i) acc = fmaf(xi[i], M[i][k], acc);
    o[(long long)k * K] = wv * acc;
  }
}

__global__ void __launch_bounds__(kThreads) dtp_forward_kernel(PlanHdr h, const uint32_t* __restrict__ blob, EdgeArgs a) {
  extern __shared__ __align__(16) uint32_t smem_raw[];
  const Smem s = carve(h, blob, smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n_tiles = (a.E + h.te - 1) / h.te;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long e0 = tile * h.te;
    __syncthreads();  // previous tile's readers are done (also covers the blob copy)
    stage_tile(h, s, a.y, e0, a.E);
    const int n_tasks = h.te * h.n_wtasks;
    for (int t = warp; t < n_tasks; t += kWarps) {
      const int te = t / h.n_wtasks;
      const long long e = e0 + te;
      if (e >= a.E) continue;
      const int2 wt = s.wtasks[t - te * h.n_wtasks];
      const PathDev& P = s.paths[wt.x];
      const float* Mp = s.M + te * h.m_size + P.m_off;
      const int u = wt.y + lane;
      EQF_DISPATCH_D(P.d1, D1, EQF_DISPATCH_D(P.d3, D3, (fwd_task<D1, D3>(h, a, P, Mp, e, u))));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// grad_w: gw[e, w_off+u] = sum_ik x_i M[i,k] g[k];   shared weights: accumulate per CTA
template <int D1, int D3>
__device__ __forceinline__ float gw_value(const PlanHdr& h, const EdgeArgs& a, const PathDev& P, const float* Mp,
                                          long long e, int u) {
  float M[D1][D3];
  load_M<D1, D3>(Mp, M);
  if (u >= P.mul) return 0.f;
  float xi[D1];
  load_x<D1>(a, P.xb, P.mul, e, u, xi);
  const int K = h.out_mul[P.og];
  const float* gp = a.g[P.og] + (e * D3) * K + P.koff + u;
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < D3; ++k) {
    const float gk = __ldg(gp + (long long)k * K);
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < D1; ++i) t = fmaf(xi[i], M[i][k], t);
    acc = fmaf(t, gk, acc);
  }
  return acc;
}

__global__ void __launch_bounds__(kThreads) dtp_grad_w_kernel(PlanHdr h, const uint32_t* __restrict__ blob, EdgeArgs a) {
  extern __shared__ __align__(16) uint32_t smem_raw[];
  const Smem s = carve(h, blob, smem_raw);
  float* wacc = s.extra;  // [w_numel] when shared
  if (a.w_shared)
    for (int i = threadIdx.x; i < h.w_numel; i += blockDim.x) wacc[i] = 0.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n_tiles = (a.E + h.te - 1) / h.te;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long e0 = tile * h.te;
    __syncthreads();
    stage_tile(h, s, a.y, e0, a.E);
    const int n_tasks = h.te * h.n_wtasks;
    for (int t = warp; t < n_tasks; t += kWarps) {
      const int te = t / h.n_wtasks;
      const long long e = e0 + te;
      if (e >= a.E) continue;
      const int2 wt = s.wtasks[t - te * h.n_wtasks];
      const PathDev& P = s.paths[wt.x];
      const float* Mp = s.M + te * h.m_size + P.m_off;
      const int u = wt.y + lane;
      float v = 0.f;
      EQF_DISPATCH_D(P.d1, D1, EQF_DISPATCH_D(P.d3, D3, (v = gw_value<D1, D3>(h, a, P, Mp, e, u))));
      if (u < P.mul) {
        if (a.w_shared) atomicAdd(wacc + P.w_off + u, v);
        else a.gw[e * h.w_numel + P.w_off + u] = v;
      }
    }
  }
  if (a.w_shared) {
    __syncthreads();
    for (int i = threadIdx.x; i < h.w_numel; i += blockDim.x) a.gw[(long long)blockIdx.x * h.w_numel + i] = wacc[i];
  }
}

// ------------------------------------------------------------------------------------------------
// grad_x (+ optionally grad_w in the same pass over g)
template <int D1, int D3, bool WITH_W>
__device__ __forceinline__ void gx_path(const PlanHdr& h, const EdgeArgs& a, const PathDev& P, const float* Mp,
                                        long long e, int u, const float (&xi)[D1], float (&acc)[D1], float* wacc) {
  float M[D1][D3];
  load_M<D1, D3>(Mp, M);
  const int K = h.out_mul[P.og];
  const float* gp = a.g[P.og] + (e * D3) * K + P.koff + u;
  float gk[D3];
#pragma unroll
  for (int k = 0; k < D3; ++k) gk[k] = __ldg(gp + (long long)k * K);
  const float wv = __ldg(a.w + (a.w_shared ? 0 : e * h.w_numel) + P.w_off + u);
  float gwv = 0.f;
#pragma unroll
  for (int i = 0; i < D1; ++i) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < D3; ++k) t = fmaf(gk[k], M[i][k], t);
    acc[i] = fmaf(wv, t, acc[i]);
    if (WITH_W) gwv = fmaf(xi[i], t, gwv);
  }
  if (WITH_W) {
    if (a.w_shared) atomicAdd(wacc + P.w_off + u, gwv);
    else a.gw[e * h.w_numel + P.w_off + u] = gwv;
  }
}

template <int D1, bool WITH_W>
__device__ __forceinline__ void gx_task(const PlanHdr& h, const EdgeArgs& a, const Smem& s, int te, long long e,
                                        int xb, int u, float* wacc) {
  const int mul = h.in1_mul[xb];
  if (u >= mul) return;  // whole-path predicate: M loads below are per-lane broadcast reads, safe to skip
  float xi[D1];
  if (WITH_W) load_x<D1>(a, xb, mul, e, u, xi);
  float acc[D1];
#pragma unroll
  for (int i = 0; i < D1; ++i) acc[i] = 0.f;
  for (int q = s.xbstart[xb]; q < s.xbstart[xb + 1]; ++q) {
    const PathDev& P = s.paths[s.xbpaths[q]];
    const float* Mp = s.M + te * h.m_size + P.m_off;
    EQF_DISPATCH_D(P.d3, D3, (gx_path<D1, D3, WITH_W>(h, a, P, Mp, e, u, xi, acc, wacc)));
  }
  float* o = a.gx[xb] + (e * D1) * mul + u;
#pragma unroll
  for (int i = 0; i < D1; ++i) o[(long long)i * mul] = acc[i];
}

template <bool WITH_W>
__global__ void __launch_bounds__(kThreads) dtp_grad_x_kernel(PlanHdr h, const uint32_t* __restrict__ blob, EdgeArgs a) {
  extern __shared__ __align__(16) uint32_t smem_raw[];
  const Smem s = carve(h, blob, smem_raw);
  float* wacc = s.extra;
  if (WITH_W && a.w_shared)
    for (int i = threadIdx.x; i < h.w_numel; i += blockDim.x) wacc[i] = 0.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n_tiles = (a.E + h.te - 1) / h.te;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long e0 = tile * h.te;
    __syncthreads();
    stage_tile(h, s, a.y, e0, a.E);
    const int n_tasks = h.te * h.n_xtasks;
    for (int t = warp; t < n_tasks; t += kWarps) {
      const int te = t / h.n_xtasks;
      const long long e = e0 + te;
      if (e >= a.E) continue;
      const int2 xt = s.xtasks[t - te * h.n_xtasks];
      const int u = xt.y + lane;
      EQF_DISPATCH_D(h.in1_d[xt.x], D1, (gx_task<D1, WITH_W>(h, a, s, te, e, xt.x, u, wacc)));
    }
  }
  if (WITH_W && a.w_shared) {
    __syncthreads();
    for (int i = threadIdx.x; i < h.w_numel; i += blockDim.x) a.gw[(long long)blockIdx.x * h.w_numel + i] = wacc[i];
  }
}

// ------------------------------------------------------------------------------------------------
// grad_y: N_p[i,k] = sum_u w x_i g_k (warp reduction) -> gy[e,j] = sum_p sum_ik C_p[i,j,k] N_p[i,k]
template <int D1, int D3>
__device__ __forceinline__ void gy_task(const PlanHdr& h, const EdgeArgs& a, const PathDev& P, float* Np,
                                        long long e, int u, int lane) {
  float xi[D1], gk[D3];
  float wv = 0.f;
#pragma unroll
  for (int i = 0; i < D1; ++i) xi[i] = 0.f;
#pragma unroll
  for (int k = 0; k < D3; ++k) gk[k] = 0.f;
  if (u < P.mul) {
    load_x<D1>(a, P.xb, P.mul, e, u, xi);
    const int K = h.out_mul[P.og];
    const float* gp = a.g[P.og] + (e * D3) * K + P.koff + u;
#pragma unroll
    for (int k = 0; k < D3; ++k) gk[k] = __ldg(gp + (long long)k * K);
    wv = __ldg(a.w + (a.w_shared ? 0 : e * h.w_numel) + P.w_off + u);
  }
#pragma unroll
  for (int i = 0; i < D1; ++i) {
    const float wx = wv * xi[i];
#pragma unroll
    for (int k = 0; k < D3; ++k) {
      const float r = warp_sum(wx * gk[k]);
      if (lane == 0) atomicAdd(Np + i * D3 + k, r);
    }
  }
}

__global__ void __launch_bounds__(kThreads) dtp_grad_y_kernel(PlanHdr h, const uint32_t* __restrict__ blob, EdgeArgs a) {
  extern __shared__ __align__(16) uint32_t smem_raw[];
  const Smem s = carve(h, blob, smem_raw);
  float* N = s.extra;  // [te][m_size]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n_tiles = (a.E + h.te - 1) / h.te;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long e0 = tile * h.te;
    __syncthreads();
    for (int i = threadIdx.x; i < h.te * h.m_size; i += blockDim.x) N[i] = 0.f;
    __syncthreads();
    const int n_tasks = h.te * h.n_wtasks;
    for (int t = warp; t < n_tasks; t += kWarps) {
      const int te = t / h.n_wtasks;
      const long long e = e0 + te;
      if (e >= a.E) continue;
      const int2 wt = s.wtasks[t - te * h.n_wtasks];
      const PathDev& P = s.paths[wt.x];
      float* Np = N + te * h.m_size + P.m_off;
      const int u = wt.y + lane;
      EQF_DISPATCH_D(P.d1, D1, EQF_DISPATCH_D(P.d3, D3, (gy_task<D1, D3>(h, a, P, Np, e, u, lane))));
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < h.te * h.d_y; idx += blockDim.x) {
      const int te = idx / h.d_y;
      const int jj = idx - te * h.d_y;
      const long long e = e0 + te;
      if (e >= a.E) continue;
      float acc = 0.f;
      for (int p = 0; p < h.n_paths; ++p) {
        const PathDev& P = s.paths[p];
        const int j = jj - P.y_off;
        if (j < 0 || j >= P.d2) continue;
        const float* c = s.cg + P.cg_off + j * P.d3;
        const float* Np = N + te * h.m_size + P.m_off;
        for (int i = 0; i < P.d1; ++i)
          for (int k = 0; k < P.d3; ++k) acc = fmaf(c[i * P.d2 * P.d3 + k], Np[i * P.d3 + k], acc);
      }
      a.gy[e * h.d_y + jj] = acc;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host launchers
static int fill_args(const EqfPlan* plan, const EqfEdgeOperands* op, long long E, EdgeArgs& a, bool need_x,
                     bool need_g, bool need_w) {
  if (plan == nullptr || op == nullptr) { set_error("null plan/operands"); return EQF_ERR_INVALID; }
  if (E < 0) { set_error("negative edge count"); return EQF_ERR_INVALID; }
  const PlanHdr& h = plan->hdr;
  for (int b = 0; b < EQF_MAX_BLOCKS; ++b) {
    a.x[b] = op->x[b]; a.x2[b] = op->x2[b]; a.g[b] = op->g[b];
    a.out[b] = nullptr; a.gx[b] = nullptr;
  }
  a.src = reinterpret_cast<const long long*>(op->src);
  a.dst = reinterpret_cast<const long long*>(op->dst);
  a.y = op->y; a.w = op->w; a.w_off = op->w_offset; a.w_shared = op->w_shared; a.gw = nullptr; a.gy = nullptr; a.E = E;
  if (E == 0) return EQF_OK;
  if (a.w_off != nullptr && !(plan->gen != nullptr && dtp_variant() == 4)) {
    set_error("w_offset is only supported by the plan-specialised kernels");
    return EQF_ERR_UNSUPPORTED;
  }
  if (a.y == nullptr) { set_error("edge_attr (y) pointer is null"); return EQF_ERR_INVALID; }
  if (need_w && a.w == nullptr) { set_error("weight pointer is null"); return EQF_ERR_INVALID; }
  if (need_x) for (int b = 0; b < h.n_in1; ++b) {
    if (a.x[b] == nullptr) { set_error("in1 block pointer is null"); return EQF_ERR_INVALID; }
    if (a.x2[b] != nullptr && a.dst == nullptr) { set_error("x2 given without dst index"); return EQF_ERR_INVALID; }
  }
  if (need_g) for (int g = 0; g < h.n_out; ++g)
    if (a.g[g] == nullptr) { set_error("output-group pointer is null"); return EQF_ERR_INVALID; }
  return ensure_device(plan);
}

static int grid_for(const EqfPlan* plan, long long E) {
  const long long n_tiles = (E + plan->hdr.te - 1) / plan->hdr.te;
  const long long cap = (long long)plan->sm_count * 8;
  return (int)(n_tiles < cap ? (n_tiles > 0 ? n_tiles : 1) : cap);
}

template <typename K>
static int set_smem(K kernel, size_t bytes) {
  if (bytes <= 48 * 1024) return EQF_OK;
  // raise the opt-in shared-memory limit once per (kernel, size), not per launch (and never inside a graph capture twice)
  static std::mutex mu;
  static std::unordered_map<const void*, size_t> configured;
  std::lock_guard<std::mutex> lock(mu);
  size_t& have = configured[reinterpret_cast<const void*>(kernel)];
  if (bytes > have) {
    int rc = check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes),
                        "cudaFuncSetAttribute(smem)");
    if (rc != EQF_OK) return rc;
    have = bytes;
  }
  return EQF_OK;
}

}  // namespace eqf

using namespace eqf;

extern "C" int eqf_plan_partial_rows(const EqfPlan* plan, int64_t n_edges) {
  if (plan == nullptr) return EQF_ERR_INVALID;
  // upper bound over the kernel generations that may write the shared-weight partial buffer
  int rows = grid_for(plan, n_edges);
  const int b = backward_v3_grid(plan, n_edges);
  if (b > rows) rows = b;
  if (plan->gen != nullptr) { const int c = plan->gen->partial_rows(plan, n_edges); if (c > rows) rows = c; }
  return rows;
}

extern "C" int eqf_dtp_forward(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges,
                               float* const* out_groups, void* stream) {
  EdgeArgs a;
  int rc = fill_args(plan, op, n_edges, a, true, false, true);
  if (rc != EQF_OK || n_edges == 0) return rc;
  for (int g = 0; g < plan->hdr.n_out; ++g) {
    if (out_groups == nullptr || out_groups[g] == nullptr) { set_error("null output group"); return EQF_ERR_INVALID; }
    a.out[g] = out_groups[g];
  }
  if (plan->gen != nullptr && dtp_variant() == 4) return plan->gen->forward(plan, a, (cudaStream_t)stream);
  if (plan->hdr.vec_ok && dtp_variant() == 3) return launch_forward_v3(plan, a, (cudaStream_t)stream);
  if (plan->hdr.vec_ok && dtp_variant() > 0)
    return launch_forward_vec(plan, a, dtp_variant() == 2 && !a.w_shared, (cudaStream_t)stream);
  const size_t smem = plan->smem_bytes;
  if ((rc = set_smem(dtp_forward_kernel, smem)) != EQF_OK) return rc;
  dtp_forward_kernel<<<grid_for(plan, n_edges), kThreads, smem, (cudaStream_t)stream>>>(plan->hdr, plan->d_blob, a);
  return check_cuda(cudaGetLastError(), "dtp_forward_kernel launch");
}

extern "C" int eqf_dtp_grad_w(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges, float* gw,
                              void* stream) {
  EdgeArgs a;
  int rc = fill_args(plan, op, n_edges, a, true, true, false);
  if (rc != EQF_OK || n_edges == 0) return rc;
  if (gw == nullptr) { set_error("null gw"); return EQF_ERR_INVALID; }
  a.gw = gw;
  const size_t smem = plan->smem_bytes;
  if ((rc = set_smem(dtp_grad_w_kernel, smem)) != EQF_OK) return rc;
  dtp_grad_w_kernel<<<grid_for(plan, n_edges), kThreads, smem, (cudaStream_t)stream>>>(plan->hdr, plan->d_blob, a);
  return check_cuda(cudaGetLastError(), "dtp_grad_w_kernel launch");
}

extern "C" int eqf_dtp_grad_x(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges,
                              float* const* gx_blocks, void* stream) {
  EdgeArgs a;
  int rc = fill_args(plan, op, n_edges, a, false, true, true);
  if (rc != EQF_OK || n_edges == 0) return rc;
  for (int b = 0; b < plan->hdr.n_in1; ++b) {
    if (gx_blocks == nullptr || gx_blocks[b] == nullptr) { set_error("null gx block"); return EQF_ERR_INVALID; }
    a.gx[b] = gx_blocks[b];
  }
  if (plan->gen != nullptr && dtp_variant() == 4) return plan->gen->backward(plan, a, false, (cudaStream_t)stream);
  if (plan->hdr.vec_ok && dtp_variant() == 3) return launch_backward_v3(plan, a, false, (cudaStream_t)stream);
  if (plan->hdr.vec_ok && dtp_variant() > 0) return launch_grad_x_vec(plan, a, false, (cudaStream_t)stream);
  const size_t smem = plan->smem_bytes;
  if ((rc = set_smem(dtp_grad_x_kernel<false>, smem)) != EQF_OK) return rc;
  dtp_grad_x_kernel<false><<<grid_for(plan, n_edges), kThreads, smem, (cudaStream_t)stream>>>(plan->hdr, plan->d_blob, a);
  return check_cuda(cudaGetLastError(), "dtp_grad_x_kernel launch");
}

extern "C" int eqf_dtp_grad_xw(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges,
                               float* const* gx_blocks, float* gw, void* stream) {
  EdgeArgs a;
  int rc = fill_args(plan, op, n_edges, a, true, true, true);
  if (rc != EQF_OK || n_edges == 0) return rc;
  if (gw == nullptr) { set_error("null gw"); return EQF_ERR_INVALID; }
  for (int b = 0; b < plan->hdr.n_in1; ++b) {
    if (gx_blocks == nullptr || gx_blocks[b] == nullptr) { set_error("null gx block"); return EQF_ERR_INVALID; }
    a.gx[b] = gx_blocks[b];
  }
  a.gw = gw;
  if (plan->gen != nullptr && dtp_variant() == 4) return plan->gen->backward(plan, a, true, (cudaStream_t)stream);
  if (plan->hdr.vec_ok && dtp_variant() == 3) return launch_backward_v3(plan, a, true, (cudaStream_t)stream);
  if (plan->hdr.vec_ok && dtp_variant() > 0) return launch_grad_x_vec(plan, a, true, (cudaStream_t)stream);
  const size_t smem = plan->smem_bytes;
  if ((rc = set_smem(dtp_grad_x_kernel<true>, smem)) != EQF_OK) return rc;
  dtp_grad_x_kernel<true><<<grid_for(plan, n_edges), kThreads, smem, (cudaStream_t)stream>>>(plan->hdr, plan->d_blob, a);
  return check_cuda(cudaGetLastError(), "dtp_grad_xw_kernel launch");
}

extern "C" int eqf_dtp_grad_y(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges, float* gy,
                              void* stream) {
  EdgeArgs a;
  int rc = fill_args(plan, op, n_edges, a, true, true, true);
  if (rc != EQF_OK || n_edges == 0) return rc;
  if (gy == nullptr) { set_error("null gy"); return EQF_ERR_INVALID; }
  a.gy = gy;
  if (plan->gen != nullptr && dtp_variant() == 4) return plan->gen->grad_y(plan, a, (cudaStream_t)stream);
  const size_t smem = plan->smem_bytes;
  if ((rc = set_smem(dtp_grad_y_kernel, smem)) != EQF_OK) return rc;
  dtp_grad_y_kernel<<<grid_for(plan, n_edges), kThreads, smem, (cudaStream_t)stream>>>(plan->hdr, plan->d_blob, a);
  return check_cuda(cudaGetLastError(), "dtp_grad_y_kernel launch");
}
