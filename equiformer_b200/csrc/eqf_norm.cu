// Per-graph equivariant norms (EquivariantGraphNorm / EquivariantInstanceNorm): see include/eqf_b200_norm.h.
//
// One CTA owns (graph g, 32-channel tile of one irreps entry) and walks the graph's nodes itself, so every statistic is
// a plain loop in a fixed order: lane ty of the 8 node lanes takes nodes ptr[g] + ty, + 8, ..., then lane 0 adds the 8
// lane sums in order.  Forward and backward each read the graph's rows two or three times (mean, centred second moment,
// apply); a graph of a few thousand atoms stays in L2 between the passes.  The CTAs stride over the graphs with a capped
// grid, so a batch of any number of graphs is one launch.
#include <cuda_runtime.h>

#include <string>

#include "eqf_b200_norm.h"

namespace eqf {

static thread_local std::string g_norm_error;
constexpr int kLanes = 8;          // node lanes per CTA
constexpr int kTile = 32;          // channels per CTA
constexpr int kMaxGraphCtas = 1024;

struct NormArgs {
  EqfSegNormLayout lay;
  const float* x[EQF_NORM_MAX_ENTRIES];
  const float* gy[EQF_NORM_MAX_ENTRIES];
  float* out[EQF_NORM_MAX_ENTRIES];  // y (forward) or gx (backward)
  const int64_t* ptr;
  int64_t G;
  const float* shift;
  const float* w;
  const float* b;
  float* mean;
  float* rstd;
  float* part;
};

static int fail(const char* msg) {
  g_norm_error = msg;
  return -1;
}

static int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return 0;
  g_norm_error = std::string(what) + ": " + cudaGetErrorString(e);
  return -2;
}

static int n_tiles(const EqfSegNormLayout& lay) {
  int t = 0;
  for (int k = 0; k < lay.n_entries; ++k) t += (lay.mul[k] + kTile - 1) / kTile;
  return t;
}

static int check_layout(const EqfSegNormLayout* lay) {
  if (!lay || lay->n_entries < 1 || lay->n_entries > EQF_NORM_MAX_ENTRIES) return fail("norm layout: 1..8 entries");
  for (int k = 0; k < lay->n_entries; ++k) {
    if (lay->mul[k] < 1 || lay->d[k] < 1) return fail("norm layout: empty entry");
    if (lay->is_scalar[k] && (lay->d[k] != 1 || lay->s_off[k] < 0)) return fail("norm layout: bad 0e entry");
  }
  return 0;
}

// entry and first channel of tile t
__device__ __forceinline__ void tile_of(const EqfSegNormLayout& lay, int t, int& k, int& c0) {
  k = 0;
  for (; k < lay.n_entries; ++k) {
    const int n = (lay.mul[k] + kTile - 1) / kTile;
    if (t < n) break;
    t -= n;
  }
  c0 = t * kTile;
}

// sum of the kLanes lane values v[ty][tx] in lane order; every thread gets the sum of its column
__device__ __forceinline__ float lane_sum(float (*red)[kTile], float v) {
  red[threadIdx.y][threadIdx.x] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < kLanes; ++j) s += red[j][threadIdx.x];
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(kTile * kLanes) norm_graph_ptr_kernel(const int64_t* batch, int64_t N, int64_t G,
                                                                         int64_t* ptr) {
  for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g <= G; g += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = N;          // first i with batch[i] >= g
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (batch[mid] < g) lo = mid + 1; else hi = mid;
    }
    ptr[g] = lo;
  }
}

__global__ void __launch_bounds__(kTile * kLanes) norm_fwd_kernel(NormArgs a) {
  __shared__ float red[kLanes][kTile];
  int k, c0;
  tile_of(a.lay, blockIdx.y, k, c0);
  const int mul = a.lay.mul[k], d = a.lay.d[k], c = c0 + threadIdx.x;
  const bool live = c < mul, scalar = a.lay.is_scalar[k] != 0;
  const int cc = live ? c : 0;
  const float* x = a.x[k];
  float* y = a.out[k];
  const float s = scalar && a.shift ? a.shift[cc] : 1.f;
  const float wc = a.w[a.lay.w_off[k] + cc];
  const float bc = scalar ? a.b[a.lay.s_off[k] + cc] : 0.f;
  const float inv_d = a.lay.component ? 1.f / d : 1.f;
  for (int64_t g = blockIdx.x; g < a.G; g += gridDim.x) {
    const int64_t n0 = a.ptr[g], n1 = a.ptr[g + 1];
    const float inv_n = n1 > n0 ? 1.f / (float)(n1 - n0) : 0.f;
    float m = 0.f;
    if (scalar) {
      float acc = 0.f;
      if (live)
        for (int64_t i = n0 + threadIdx.y; i < n1; i += kLanes) acc += x[i * mul + c];
      m = lane_sum(red, acc) * inv_n;
    }
    const float msh = s * m;
    float acc = 0.f;
    if (live)
      for (int64_t i = n0 + threadIdx.y; i < n1; i += kLanes)
        for (int j = 0; j < d; ++j) {
          const float z = x[(i * d + j) * mul + c] - msh;
          acc = fmaf(z, z, acc);
        }
    const float v = lane_sum(red, acc) * inv_n * inv_d;
    const float r = 1.f / sqrtf(v + a.lay.eps);
    const float sc = r * wc;
    if (!live) continue;
    if (threadIdx.y == 0) {
      a.rstd[g * a.lay.n_w + a.lay.w_off[k] + c] = r;
      if (scalar) a.mean[g * a.lay.n_s + a.lay.s_off[k] + c] = m;
    }
    for (int64_t i = n0 + threadIdx.y; i < n1; i += kLanes)
      for (int j = 0; j < d; ++j) {
        const int64_t o = (i * d + j) * mul + c;
        y[o] = fmaf(x[o] - msh, sc, bc);
      }
  }
}

// y = z r w + b with z = x - s m (0e) or x, r = (v + eps)^-1/2, v = mean_i |z_i|^2 / D:
//   dL/dz_i = gy_i r w - c1 z_i,  c1 = r^3 w S1 / (n D),  S1 = sum_i gy_i . z_i
//   0e:  dL/dx_i = dL/dz_i - (s / n) sum_j dL/dz_j,  d shift = -m sum_j dL/dz_j
//   d w = r S1,  d b = sum_i gy_i
__global__ void __launch_bounds__(kTile * kLanes) norm_bwd_kernel(NormArgs a) {
  __shared__ float red[kLanes][kTile];
  int k, c0;
  tile_of(a.lay, blockIdx.y, k, c0);
  const int mul = a.lay.mul[k], d = a.lay.d[k], c = c0 + threadIdx.x;
  const bool live = c < mul, scalar = a.lay.is_scalar[k] != 0;
  const int cc = live ? c : 0;
  const float* x = a.x[k];
  const float* gy = a.gy[k];
  float* gx = a.out[k];
  const float s = scalar && a.shift ? a.shift[cc] : 1.f;
  const float wc = a.w[a.lay.w_off[k] + cc];
  const float inv_d = a.lay.component ? 1.f / d : 1.f;
  const int cols = a.lay.n_w + 2 * a.lay.n_s;
  for (int64_t g = blockIdx.x; g < a.G; g += gridDim.x) {
    const int64_t n0 = a.ptr[g], n1 = a.ptr[g + 1];
    const float inv_n = n1 > n0 ? 1.f / (float)(n1 - n0) : 0.f;
    const float r = live ? a.rstd[g * a.lay.n_w + a.lay.w_off[k] + c] : 0.f;
    const float m = scalar && live ? a.mean[g * a.lay.n_s + a.lay.s_off[k] + c] : 0.f;
    const float msh = s * m;
    float s0 = 0.f, s1 = 0.f, sz = 0.f;
    if (live)
      for (int64_t i = n0 + threadIdx.y; i < n1; i += kLanes)
        for (int j = 0; j < d; ++j) {
          const int64_t o = (i * d + j) * mul + c;
          const float z = x[o] - msh, t = gy[o];
          s0 += t;
          s1 = fmaf(t, z, s1);
          sz += z;
        }
    s0 = lane_sum(red, s0);
    s1 = lane_sum(red, s1);
    sz = scalar ? lane_sum(red, sz) : 0.f;
    if (!live) continue;
    const float sc = r * wc;
    const float c1 = r * r * r * wc * s1 * inv_n * inv_d;
    const float sum_dz = sc * s0 - c1 * sz;             // 0e entries only
    const float corr = scalar ? s * inv_n * sum_dz : 0.f;
    if (threadIdx.y == 0) {
      float* p = a.part + g * cols;
      p[a.lay.w_off[k] + c] = r * s1;
      if (scalar) {
        p[a.lay.n_w + a.lay.s_off[k] + c] = s0;
        p[a.lay.n_w + a.lay.n_s + a.lay.s_off[k] + c] = -m * sum_dz;
      }
    }
    for (int64_t i = n0 + threadIdx.y; i < n1; i += kLanes)
      for (int j = 0; j < d; ++j) {
        const int64_t o = (i * d + j) * mul + c;
        gx[o] = gy[o] * sc - c1 * (x[o] - msh) - corr;
      }
  }
}

// out[col] = sum over g = 0 .. G-1 of part[g][col], in that order
__global__ void __launch_bounds__(256) norm_param_reduce_kernel(const float* part, int64_t G, int cols, float* out) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= cols) return;
  float acc = 0.f;
  for (int64_t g = 0; g < G; ++g) acc += part[g * cols + col];
  out[col] = acc;
}

static int fill(const EqfSegNormLayout* lay, const float* const* x_blocks, int64_t n_graphs, const int64_t* graph_ptr,
         const float* w, NormArgs& a) {
  int rc = check_layout(lay);
  if (rc) return rc;
  if (!x_blocks || !graph_ptr || !w) return fail("eqf_norm: null pointer");
  a = NormArgs{};
  a.lay = *lay;
  a.ptr = graph_ptr;
  a.G = n_graphs;
  a.w = w;
  for (int k = 0; k < lay->n_entries; ++k) {
    if (!x_blocks[k]) return fail("eqf_norm: null block");
    a.x[k] = x_blocks[k];
  }
  return 0;
}

static dim3 grid(const EqfSegNormLayout& lay, int64_t G) {
  return dim3((unsigned)(G < kMaxGraphCtas ? G : kMaxGraphCtas), (unsigned)n_tiles(lay));
}

}  // namespace eqf

using namespace eqf;

extern "C" const char* eqf_last_error(void) { return g_norm_error.c_str(); }

extern "C" int eqf_norm_graph_ptr(const int64_t* batch, int64_t N, int64_t n_graphs, int64_t* graph_ptr, void* stream) {
  if (n_graphs < 0 || N < 0 || !graph_ptr || (N > 0 && !batch)) return fail("eqf_norm_graph_ptr: bad arguments");
  const int64_t blocks = (n_graphs + 1 + 255) / 256;
  norm_graph_ptr_kernel<<<(unsigned)(blocks < 1024 ? blocks : 1024), 256, 0, (cudaStream_t)stream>>>(batch, N, n_graphs,
                                                                                                      graph_ptr);
  return check_launch("norm_graph_ptr_kernel launch");
}

extern "C" int eqf_norm_fwd(const EqfSegNormLayout* lay, const float* const* x_blocks, const int64_t* graph_ptr,
                            int64_t n_graphs, const float* shift, const float* w, const float* b, float* const* y_blocks,
                            float* mean, float* rstd, void* stream) {
  NormArgs a;
  int rc = fill(lay, x_blocks, n_graphs, graph_ptr, w, a);
  if (rc || n_graphs == 0) return rc;
  if (!y_blocks || !rstd || (lay->n_s > 0 && (!b || !mean))) return fail("eqf_norm_fwd: null pointer");
  a.shift = shift;
  a.b = b;
  a.mean = mean;
  a.rstd = rstd;
  for (int k = 0; k < lay->n_entries; ++k) {
    if (!y_blocks[k]) return fail("eqf_norm_fwd: null output block");
    a.out[k] = y_blocks[k];
  }
  norm_fwd_kernel<<<grid(*lay, n_graphs), dim3(kTile, kLanes), 0, (cudaStream_t)stream>>>(a);
  return check_launch("norm_fwd_kernel launch");
}

extern "C" int eqf_norm_bwd(const EqfSegNormLayout* lay, const float* const* x_blocks, const float* const* gy_blocks,
                            const int64_t* graph_ptr, int64_t n_graphs, const float* shift, const float* w,
                            const float* mean, const float* rstd, float* const* gx_blocks, float* part, void* stream) {
  NormArgs a;
  int rc = fill(lay, x_blocks, n_graphs, graph_ptr, w, a);
  if (rc || n_graphs == 0) return rc;
  if (!gy_blocks || !gx_blocks || !rstd || !part || (lay->n_s > 0 && !mean)) return fail("eqf_norm_bwd: null pointer");
  a.shift = shift;
  a.mean = const_cast<float*>(mean);
  a.rstd = const_cast<float*>(rstd);
  a.part = part;
  for (int k = 0; k < lay->n_entries; ++k) {
    if (!gy_blocks[k] || !gx_blocks[k]) return fail("eqf_norm_bwd: null block");
    a.gy[k] = gy_blocks[k];
    a.out[k] = gx_blocks[k];
  }
  norm_bwd_kernel<<<grid(*lay, n_graphs), dim3(kTile, kLanes), 0, (cudaStream_t)stream>>>(a);
  return check_launch("norm_bwd_kernel launch");
}

extern "C" int eqf_norm_param_reduce(const float* part, int64_t n_graphs, int32_t cols, float* out, void* stream) {
  if (cols <= 0 || n_graphs < 0 || !out || (n_graphs > 0 && !part)) return fail("eqf_norm_param_reduce: bad arguments");
  norm_param_reduce_kernel<<<(cols + 255) / 256, 256, 0, (cudaStream_t)stream>>>(part, n_graphs, cols, out);
  return check_launch("norm_param_reduce_kernel launch");
}
