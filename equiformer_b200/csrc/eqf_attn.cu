// eqf_attn.cu - segmented softmax and attention-weighted aggregation over destination-sorted edges.
//
// Reference work replaced (nets/graph_attention_transformer.py):
//   :508      torch_geometric.utils.softmax(alpha, edge_dst)   -> seg_softmax_kernel
//   :512-513  value * alpha ; torch_scatter.scatter(.., edge_dst) -> aggregate_kernel (no atomics: the
//             edge list is sorted by destination, each output row is owned by one warp)
// plus the two transposes that autograd needs (edge_dot, edge_scale).  aggregate / edge_dot /
// edge_scale are the three partial derivatives of the trilinear form
//     T(alpha, V, G) = sum_e sum_j alpha[e, head(j)] V[e, j] G[dst[e], j]
// so the family is closed under differentiation (double backward for MD17 forces).
//
// All three are HBM streaming kernels: aggregate reads V once (4*D_v bytes/edge), lanes run over
// the channel-innermost planar layout.
#include <math_constants.h>

#include "eqf_common.cuh"

namespace eqf {

struct HeadArgs {
  int n_groups, n_heads;
  int d[EQF_MAX_BLOCKS];
  int C[EQF_MAX_BLOCKS];
  int rowlen[EQF_MAX_BLOCKS];      // d*C
  int chunk_start[EQF_MAX_BLOCKS + 1];  // prefix sum of ceil(rowlen/32)
  const float* V[EQF_MAX_BLOCKS];
  const float* G[EQF_MAX_BLOCKS];
  float* out[EQF_MAX_BLOCKS];
};

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_add(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// one warp per destination node; all heads
__global__ void __launch_bounds__(256) seg_softmax_kernel(const float* __restrict__ z, const long long* __restrict__ row_ptr,
                                                          long long n_nodes, int H, float* __restrict__ alpha) {
  const long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= n_nodes) return;
  const int lane = threadIdx.x & 31;
  const long long r0 = row_ptr[t], r1 = row_ptr[t + 1];
  for (int h = 0; h < H; ++h) {
    float m = -CUDART_INF_F;
    for (long long e = r0 + lane; e < r1; e += 32) m = fmaxf(m, __ldg(z + e * H + h));
    m = warp_max(m);
    float s = 0.f;
    for (long long e = r0 + lane; e < r1; e += 32) s += expf(__ldg(z + e * H + h) - m);
    s = warp_add(s);
    const float inv = 1.f / (s + 1e-16f);
    for (long long e = r0 + lane; e < r1; e += 32) alpha[e * H + h] = expf(__ldg(z + e * H + h) - m) * inv;
  }
}

// backward of the segment softmax: gz_e = alpha_e (ga_e - sum_{f in seg(e)} alpha_f ga_f); one warp per destination node
// (the eager version is a multiply, an index_add into [N, H], a gather back to [E, H], a multiply and a subtract)
__global__ void __launch_bounds__(256) seg_softmax_bwd_kernel(const float* __restrict__ alpha, const float* __restrict__ ga,
                                                              const long long* __restrict__ row_ptr, long long n_nodes, int H,
                                                              float* __restrict__ gz) {
  const long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= n_nodes) return;
  const int lane = threadIdx.x & 31;
  const long long r0 = row_ptr[t], r1 = row_ptr[t + 1];
  for (int h = 0; h < H; ++h) {
    float s = 0.f;
    for (long long e = r0 + lane; e < r1; e += 32) s += __ldg(alpha + e * H + h) * __ldg(ga + e * H + h);
    s = warp_add(s);
    for (long long e = r0 + lane; e < r1; e += 32) {
      const float a = __ldg(alpha + e * H + h);
      gz[e * H + h] = a * (__ldg(ga + e * H + h) - s);
    }
  }
}

__device__ __forceinline__ int find_group(const HeadArgs& a, int chunk) {
  int g = 0;
  while (g + 1 < a.n_groups && chunk >= a.chunk_start[g + 1]) ++g;
  return g;
}

// one warp per (node, 32-column chunk)
// `perm` (optional): segment position -> edge id, for reducing by an index the edge list is NOT sorted by
// (the CSC side: gradients of the gathered source rows).
__global__ void __launch_bounds__(256) aggregate_kernel(HeadArgs a, const float* __restrict__ alpha,
                                                        const long long* __restrict__ row_ptr,
                                                        const long long* __restrict__ perm, long long n_nodes) {
  const int n_chunks = a.chunk_start[a.n_groups];
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= n_nodes * n_chunks) return;
  const long long t = wid / n_chunks;
  const int chunk = (int)(wid - t * n_chunks);
  const int g = find_group(a, chunk);
  const int j = (chunk - a.chunk_start[g]) * 32 + (threadIdx.x & 31);
  const int rowlen = a.rowlen[g];
  if (j >= rowlen) return;
  const int c = j % a.C[g];
  const int h = c / (a.C[g] / a.n_heads);
  const long long r0 = row_ptr[t], r1 = row_ptr[t + 1];
  const float* __restrict__ v = a.V[g] + j;
  float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
  long long e = r0;
  if (perm != nullptr) {
    const int H = a.n_heads;
    for (; e < r1; ++e) {
      const long long id = __ldg(perm + e);
      const float al = alpha ? __ldg(alpha + id * H + h) : 1.f;
      acc0 = fmaf(al, __ldg(v + id * rowlen), acc0);
    }
  } else if (alpha != nullptr) {
    const float* __restrict__ al = alpha + h;
    const int H = a.n_heads;
    for (; e + 3 < r1; e += 4) {
      const float v0 = __ldg(v + e * rowlen), v1 = __ldg(v + (e + 1) * rowlen);
      const float v2 = __ldg(v + (e + 2) * rowlen), v3 = __ldg(v + (e + 3) * rowlen);
      acc0 = fmaf(__ldg(al + e * H), v0, acc0);
      acc1 = fmaf(__ldg(al + (e + 1) * H), v1, acc1);
      acc2 = fmaf(__ldg(al + (e + 2) * H), v2, acc2);
      acc3 = fmaf(__ldg(al + (e + 3) * H), v3, acc3);
    }
    for (; e < r1; ++e) acc0 = fmaf(__ldg(al + e * H), __ldg(v + e * rowlen), acc0);
  } else {
    for (; e + 3 < r1; e += 4) {
      acc0 += __ldg(v + e * rowlen);
      acc1 += __ldg(v + (e + 1) * rowlen);
      acc2 += __ldg(v + (e + 2) * rowlen);
      acc3 += __ldg(v + (e + 3) * rowlen);
    }
    for (; e < r1; ++e) acc0 += __ldg(v + e * rowlen);
  }
  a.out[g][t * rowlen + j] = (acc0 + acc1) + (acc2 + acc3);
}

// one warp per edge: galpha[e,h] = sum_{j in head h} V[e,j] G[dst[e],j]
__global__ void __launch_bounds__(256) edge_dot_kernel(HeadArgs a, const long long* __restrict__ dst, long long n_edges,
                                                       float* __restrict__ galpha) {
  const long long e = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (e >= n_edges) return;
  const int lane = threadIdx.x & 31;
  const long long t = dst[e];
  float acc[EQF_MAX_HEADS];
#pragma unroll
  for (int h = 0; h < EQF_MAX_HEADS; ++h) acc[h] = 0.f;
  for (int g = 0; g < a.n_groups; ++g) {
    const int rowlen = a.rowlen[g], C = a.C[g], ch = C / a.n_heads;
    const float* __restrict__ v = a.V[g] + e * rowlen;
    const float* __restrict__ gg = a.G[g] + t * rowlen;
    for (int j = lane; j < rowlen; j += 32) {
      const float p = __ldg(v + j) * __ldg(gg + j);
      const int h = (j % C) / ch;
#pragma unroll
      for (int q = 0; q < EQF_MAX_HEADS; ++q) acc[q] += (q == h) ? p : 0.f;
    }
  }
#pragma unroll
  for (int q = 0; q < EQF_MAX_HEADS; ++q) {
    if (q < a.n_heads) {
      const float r = warp_add(acc[q]);
      if (lane == 0) galpha[e * a.n_heads + q] = r;
    }
  }
}

// elementwise: out[g][e,j] = alpha[e,head(j)] * G[g][dst[e],j]; grid.y = group
__global__ void __launch_bounds__(256) edge_scale_kernel(HeadArgs a, const float* __restrict__ alpha,
                                                         const long long* __restrict__ dst, long long n_edges) {
  const int g = blockIdx.y;
  const int rowlen = a.rowlen[g];
  const long long total = n_edges * rowlen;
  const int C = a.C[g], ch = C / a.n_heads, H = a.n_heads;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long e = idx / rowlen;
    const int j = (int)(idx - e * rowlen);
    const long long t = dst[e];
    float v = __ldg(a.G[g] + t * rowlen + j);
    if (alpha != nullptr) v *= __ldg(alpha + e * H + (j % C) / ch);
    a.out[g][idx] = v;
  }
}

// ------------------------------------------------------------------------------------------------ 128-bit variants
// Used when every group has rowlen % 4 == 0 and (C / H) % 4 == 0 (all shipped configs): a lane owns four consecutive
// channels (same head), a warp instruction moves 512 contiguous bytes.
__device__ __forceinline__ float4 ldv(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// one warp per (node, 128-column chunk)
__global__ void __launch_bounds__(256) aggregate_vec_kernel(HeadArgs a, const float* __restrict__ alpha,
                                                            const long long* __restrict__ row_ptr,
                                                            const long long* __restrict__ perm, long long n_nodes) {
  const int n_chunks = a.chunk_start[a.n_groups];   // here: chunks of 128 columns
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= n_nodes * n_chunks) return;
  const long long t = wid / n_chunks;
  const int chunk = (int)(wid - t * n_chunks);
  const int g = find_group(a, chunk);
  const int j = (chunk - a.chunk_start[g]) * 128 + (threadIdx.x & 31) * 4;
  const int rowlen = a.rowlen[g];
  if (j >= rowlen) return;
  const int H = a.n_heads;
  const int h = (j % a.C[g]) / (a.C[g] / H);
  const long long r0 = row_ptr[t], r1 = row_ptr[t + 1];
  const float* __restrict__ v = a.V[g] + j;
  float4 acc0 = make_float4(0.f, 0.f, 0.f, 0.f), acc1 = acc0;
  long long e = r0;
  for (; e + 1 < r1; e += 2) {
    const long long i0 = perm ? __ldg(perm + e) : e, i1 = perm ? __ldg(perm + e + 1) : e + 1;
    const float a0 = alpha ? __ldg(alpha + i0 * H + h) : 1.f, a1 = alpha ? __ldg(alpha + i1 * H + h) : 1.f;
    const float4 v0 = ldv(v + i0 * rowlen), v1 = ldv(v + i1 * rowlen);
    acc0.x = fmaf(a0, v0.x, acc0.x); acc0.y = fmaf(a0, v0.y, acc0.y); acc0.z = fmaf(a0, v0.z, acc0.z); acc0.w = fmaf(a0, v0.w, acc0.w);
    acc1.x = fmaf(a1, v1.x, acc1.x); acc1.y = fmaf(a1, v1.y, acc1.y); acc1.z = fmaf(a1, v1.z, acc1.z); acc1.w = fmaf(a1, v1.w, acc1.w);
  }
  if (e < r1) {
    const long long i0 = perm ? __ldg(perm + e) : e;
    const float a0 = alpha ? __ldg(alpha + i0 * H + h) : 1.f;
    const float4 v0 = ldv(v + i0 * rowlen);
    acc0.x = fmaf(a0, v0.x, acc0.x); acc0.y = fmaf(a0, v0.y, acc0.y); acc0.z = fmaf(a0, v0.z, acc0.z); acc0.w = fmaf(a0, v0.w, acc0.w);
  }
  *reinterpret_cast<float4*>(a.out[g] + t * rowlen + j) =
      make_float4(acc0.x + acc1.x, acc0.y + acc1.y, acc0.z + acc1.z, acc0.w + acc1.w);
}

// K2: segment softmax AND attention-weighted aggregation in one pass (ref :508 + :512-513): one warp per (node, 128-column
// chunk) first reduces its head's logits over the destination segment (max, then sum of exponentials - the segment is a
// few dozen edges of one L1-resident row range, every lane of a head reads the same addresses), then accumulates
// alpha_e V_e with alpha_e = exp(z_e - max) / (sum + 1e-16) computed on the fly; alpha[E, H] is written once (by the lanes
// that own the first channel of each head in the 0e group) because the backward needs it.
__global__ void __launch_bounds__(256) softmax_aggregate_vec_kernel(HeadArgs a, const float* __restrict__ z,
                                                                    const long long* __restrict__ row_ptr, long long n_nodes,
                                                                    float* __restrict__ alpha_out) {
  const int n_chunks = a.chunk_start[a.n_groups];
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= n_nodes * n_chunks) return;
  const long long t = wid / n_chunks;
  const int chunk = (int)(wid - t * n_chunks);
  const int g = find_group(a, chunk);
  const int j = (chunk - a.chunk_start[g]) * 128 + (threadIdx.x & 31) * 4;
  const int rowlen = a.rowlen[g];
  if (j >= rowlen) return;
  const int H = a.n_heads;
  const int per_head = a.C[g] / H;
  const int h = (j % a.C[g]) / per_head;
  const long long r0 = row_ptr[t], r1 = row_ptr[t + 1];
  float m = -CUDART_INF_F;
  for (long long e = r0; e < r1; ++e) m = fmaxf(m, __ldg(z + e * H + h));
  float sum = 0.f;
  for (long long e = r0; e < r1; ++e) sum += expf(__ldg(z + e * H + h) - m);
  const float inv = 1.f / (sum + 1e-16f);
  const bool writer = alpha_out != nullptr && g == 0 && j < a.C[0] && (j % per_head) == 0;
  const float* __restrict__ v = a.V[g] + j;
  float4 acc0 = make_float4(0.f, 0.f, 0.f, 0.f), acc1 = acc0;
  long long e = r0;
  for (; e + 1 < r1; e += 2) {
    const float a0 = expf(__ldg(z + e * H + h) - m) * inv, a1 = expf(__ldg(z + (e + 1) * H + h) - m) * inv;
    const float4 v0 = ldv(v + e * rowlen), v1 = ldv(v + (e + 1) * rowlen);
    if (writer) { alpha_out[e * H + h] = a0; alpha_out[(e + 1) * H + h] = a1; }
    acc0.x = fmaf(a0, v0.x, acc0.x); acc0.y = fmaf(a0, v0.y, acc0.y); acc0.z = fmaf(a0, v0.z, acc0.z); acc0.w = fmaf(a0, v0.w, acc0.w);
    acc1.x = fmaf(a1, v1.x, acc1.x); acc1.y = fmaf(a1, v1.y, acc1.y); acc1.z = fmaf(a1, v1.z, acc1.z); acc1.w = fmaf(a1, v1.w, acc1.w);
  }
  if (e < r1) {
    const float a0 = expf(__ldg(z + e * H + h) - m) * inv;
    const float4 v0 = ldv(v + e * rowlen);
    if (writer) alpha_out[e * H + h] = a0;
    acc0.x = fmaf(a0, v0.x, acc0.x); acc0.y = fmaf(a0, v0.y, acc0.y); acc0.z = fmaf(a0, v0.z, acc0.z); acc0.w = fmaf(a0, v0.w, acc0.w);
  }
  *reinterpret_cast<float4*>(a.out[g] + t * rowlen + j) =
      make_float4(acc0.x + acc1.x, acc0.y + acc1.y, acc0.z + acc1.z, acc0.w + acc1.w);
}

// one warp per edge, H accumulators per lane
template <int H>
__global__ void __launch_bounds__(256) edge_dot_vec_kernel(HeadArgs a, const long long* __restrict__ dst, long long n_edges,
                                                           float* __restrict__ galpha) {
  const long long e = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (e >= n_edges) return;
  const int lane = threadIdx.x & 31;
  const long long t = dst[e];
  float acc[H];
#pragma unroll
  for (int h = 0; h < H; ++h) acc[h] = 0.f;
  for (int g = 0; g < a.n_groups; ++g) {
    const int rowlen = a.rowlen[g], C = a.C[g], ch = C / H;
    const float* __restrict__ v = a.V[g] + e * rowlen;
    const float* __restrict__ gg = a.G[g] + t * rowlen;
    for (int j = lane * 4; j < rowlen; j += 128) {
      const float4 x = ldv(v + j), y = ldv(gg + j);
      const float p = x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
      const int h = (j % C) / ch;
#pragma unroll
      for (int q = 0; q < H; ++q) acc[q] += (q == h) ? p : 0.f;
    }
  }
#pragma unroll
  for (int q = 0; q < H; ++q) {
    const float r = warp_add(acc[q]);
    if (lane == 0) galpha[e * H + q] = r;
  }
}

// one warp per edge: out[g][e, j] = alpha[e, head(j)] * G[g][dst[e], j]
__global__ void __launch_bounds__(256) edge_scale_vec_kernel(HeadArgs a, const float* __restrict__ alpha,
                                                             const long long* __restrict__ dst, long long n_edges) {
  const int lane = threadIdx.x & 31;
  const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long e = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); e < n_edges; e += n_warps) {
    const long long t = dst[e];
    for (int g = 0; g < a.n_groups; ++g) {
      const int rowlen = a.rowlen[g], C = a.C[g], ch = C / a.n_heads;
      const float* __restrict__ gg = a.G[g] + t * rowlen;
      float* __restrict__ o = a.out[g] + e * rowlen;
      for (int j = lane * 4; j < rowlen; j += 128) {
        float4 v = ldv(gg + j);
        if (alpha != nullptr) {
          const float s = __ldg(alpha + e * a.n_heads + (j % C) / ch);
          v.x *= s; v.y *= s; v.z *= s; v.w *= s;
        }
        *reinterpret_cast<float4*>(o + j) = v;
      }
    }
  }
}

static bool vec_ok(const HeadArgs& a) {
  for (int g = 0; g < a.n_groups; ++g)
    if (a.rowlen[g] % 4 != 0 || (a.C[g] / a.n_heads) % 4 != 0) return false;
  return true;
}

static int fill_head_args(const EqfHeadLayout* lay, HeadArgs& a) {
  if (lay == nullptr) { set_error("null head layout"); return EQF_ERR_INVALID; }
  if (lay->n_groups < 1 || lay->n_groups > EQF_MAX_BLOCKS) { set_error("bad n_groups"); return EQF_ERR_INVALID; }
  if (lay->n_heads < 1 || lay->n_heads > EQF_MAX_HEADS) { set_error("bad n_heads"); return EQF_ERR_INVALID; }
  a.n_groups = lay->n_groups; a.n_heads = lay->n_heads;
  a.chunk_start[0] = 0;
  for (int g = 0; g < EQF_MAX_BLOCKS; ++g) { a.V[g] = nullptr; a.G[g] = nullptr; a.out[g] = nullptr; }
  for (int g = 0; g < lay->n_groups; ++g) {
    if (lay->d[g] < 1 || lay->C[g] < 1 || lay->C[g] % lay->n_heads != 0) {
      set_error("group channels must be a positive multiple of n_heads"); return EQF_ERR_INVALID;
    }
    a.d[g] = lay->d[g]; a.C[g] = lay->C[g]; a.rowlen[g] = lay->d[g] * lay->C[g];
    a.chunk_start[g + 1] = a.chunk_start[g] + (a.rowlen[g] + 31) / 32;
  }
  return EQF_OK;
}

}  // namespace eqf

using namespace eqf;

extern "C" int eqf_seg_softmax(const float* z, const int64_t* row_ptr, int64_t n_nodes, int32_t n_heads,
                               float* alpha, void* stream) {
  if (n_nodes == 0) return EQF_OK;
  if (z == nullptr || row_ptr == nullptr || alpha == nullptr || n_heads < 1) {
    set_error("eqf_seg_softmax: null pointer or bad head count"); return EQF_ERR_INVALID;
  }
  const int wpb = 8;
  const long long blocks = (n_nodes + wpb - 1) / wpb;
  seg_softmax_kernel<<<(unsigned)blocks, wpb * 32, 0, (cudaStream_t)stream>>>(
      z, reinterpret_cast<const long long*>(row_ptr), n_nodes, n_heads, alpha);
  return check_cuda(cudaGetLastError(), "seg_softmax_kernel launch");
}

extern "C" int eqf_seg_softmax_bwd(const float* alpha, const float* ga, const int64_t* row_ptr, int64_t n_nodes,
                                   int32_t n_heads, float* gz, void* stream) {
  if (n_nodes == 0) return EQF_OK;
  if (!alpha || !ga || !row_ptr || !gz || n_heads < 1) { set_error("eqf_seg_softmax_bwd: bad arguments"); return EQF_ERR_INVALID; }
  const int wpb = 8;
  const long long blocks = (n_nodes + wpb - 1) / wpb;
  seg_softmax_bwd_kernel<<<(unsigned)blocks, wpb * 32, 0, (cudaStream_t)stream>>>(
      alpha, ga, reinterpret_cast<const long long*>(row_ptr), n_nodes, n_heads, gz);
  return check_cuda(cudaGetLastError(), "seg_softmax_bwd_kernel launch");
}

extern "C" int eqf_attn_aggregate(const EqfHeadLayout* lay, const float* alpha, const float* const* V,
                                  const int64_t* row_ptr, const int64_t* perm, int64_t n_nodes, float* const* out,
                                  void* stream) {
  HeadArgs a;
  int rc = fill_head_args(lay, a);
  if (rc != EQF_OK || n_nodes == 0) return rc;
  if (V == nullptr || out == nullptr || row_ptr == nullptr) { set_error("eqf_attn_aggregate: null pointer"); return EQF_ERR_INVALID; }
  for (int g = 0; g < a.n_groups; ++g) {
    if (V[g] == nullptr || out[g] == nullptr) { set_error("eqf_attn_aggregate: null group"); return EQF_ERR_INVALID; }
    a.V[g] = V[g]; a.out[g] = out[g];
  }
  const int wpb = 8;
  if (vec_ok(a)) {
    for (int g = 0; g < a.n_groups; ++g) a.chunk_start[g + 1] = a.chunk_start[g] + (a.rowlen[g] + 127) / 128;
    const long long warps = n_nodes * a.chunk_start[a.n_groups];
    aggregate_vec_kernel<<<(unsigned)((warps + wpb - 1) / wpb), wpb * 32, 0, (cudaStream_t)stream>>>(
        a, alpha, reinterpret_cast<const long long*>(row_ptr), reinterpret_cast<const long long*>(perm), n_nodes);
    return check_cuda(cudaGetLastError(), "aggregate_vec_kernel launch");
  }
  const long long warps = n_nodes * a.chunk_start[a.n_groups];
  const long long blocks = (warps + wpb - 1) / wpb;
  aggregate_kernel<<<(unsigned)blocks, wpb * 32, 0, (cudaStream_t)stream>>>(
      a, alpha, reinterpret_cast<const long long*>(row_ptr), reinterpret_cast<const long long*>(perm), n_nodes);
  return check_cuda(cudaGetLastError(), "aggregate_kernel launch");
}

// out[g][t] = sum_{e -> t} softmax_t(z)[e, head] V[g][e]  and  alpha[E, H] = the softmax (PyG semantics) in ONE launch.
// Needs the float4 layout (every group's channels % 4 == 0), a leading group with one component (0e) whose channels per
// head are a multiple of 4 (it is the one whose lanes write alpha); EQF_ERR_UNSUPPORTED otherwise.
extern "C" int eqf_attn_softmax_aggregate(const EqfHeadLayout* lay, const float* z, const float* const* V,
                                          const int64_t* row_ptr, int64_t n_nodes, float* const* out, float* alpha,
                                          void* stream) {
  HeadArgs a;
  int rc = fill_head_args(lay, a);
  if (rc != EQF_OK || n_nodes == 0) return rc;
  if (z == nullptr || V == nullptr || out == nullptr || row_ptr == nullptr || alpha == nullptr) {
    set_error("eqf_attn_softmax_aggregate: null pointer"); return EQF_ERR_INVALID;
  }
  for (int g = 0; g < a.n_groups; ++g) {
    if (V[g] == nullptr || out[g] == nullptr) { set_error("eqf_attn_softmax_aggregate: null group"); return EQF_ERR_INVALID; }
    a.V[g] = V[g]; a.out[g] = out[g];
  }
  if (!vec_ok(a) || a.d[0] != 1 || (a.C[0] / a.n_heads) % 4 != 0) {
    set_error("eqf_attn_softmax_aggregate: layout not supported by the fused kernel"); return EQF_ERR_UNSUPPORTED;
  }
  for (int g = 0; g < a.n_groups; ++g) a.chunk_start[g + 1] = a.chunk_start[g] + (a.rowlen[g] + 127) / 128;
  const int wpb = 8;
  const long long warps = n_nodes * a.chunk_start[a.n_groups];
  softmax_aggregate_vec_kernel<<<(unsigned)((warps + wpb - 1) / wpb), wpb * 32, 0, (cudaStream_t)stream>>>(
      a, z, reinterpret_cast<const long long*>(row_ptr), n_nodes, alpha);
  return check_cuda(cudaGetLastError(), "softmax_aggregate_vec_kernel launch");
}

extern "C" int eqf_attn_edge_dot(const EqfHeadLayout* lay, const float* const* V, const float* const* G,
                                 const int64_t* dst, int64_t n_edges, float* galpha, void* stream) {
  HeadArgs a;
  int rc = fill_head_args(lay, a);
  if (rc != EQF_OK || n_edges == 0) return rc;
  if (V == nullptr || G == nullptr || dst == nullptr || galpha == nullptr) { set_error("eqf_attn_edge_dot: null pointer"); return EQF_ERR_INVALID; }
  for (int g = 0; g < a.n_groups; ++g) {
    if (V[g] == nullptr || G[g] == nullptr) { set_error("eqf_attn_edge_dot: null group"); return EQF_ERR_INVALID; }
    a.V[g] = V[g]; a.G[g] = G[g];
  }
  const int wpb = 8;
  const long long blocks = (n_edges + wpb - 1) / wpb;
  const long long* d = reinterpret_cast<const long long*>(dst);
  cudaStream_t st = (cudaStream_t)stream;
  if (vec_ok(a) && (a.n_heads == 1 || a.n_heads == 2 || a.n_heads == 4 || a.n_heads == 8 || a.n_heads == 16)) {
    switch (a.n_heads) {
      case 1: edge_dot_vec_kernel<1><<<(unsigned)blocks, wpb * 32, 0, st>>>(a, d, n_edges, galpha); break;
      case 2: edge_dot_vec_kernel<2><<<(unsigned)blocks, wpb * 32, 0, st>>>(a, d, n_edges, galpha); break;
      case 4: edge_dot_vec_kernel<4><<<(unsigned)blocks, wpb * 32, 0, st>>>(a, d, n_edges, galpha); break;
      case 8: edge_dot_vec_kernel<8><<<(unsigned)blocks, wpb * 32, 0, st>>>(a, d, n_edges, galpha); break;
      default: edge_dot_vec_kernel<16><<<(unsigned)blocks, wpb * 32, 0, st>>>(a, d, n_edges, galpha); break;
    }
    return check_cuda(cudaGetLastError(), "edge_dot_vec_kernel launch");
  }
  edge_dot_kernel<<<(unsigned)blocks, wpb * 32, 0, st>>>(a, d, n_edges, galpha);
  return check_cuda(cudaGetLastError(), "edge_dot_kernel launch");
}

extern "C" int eqf_attn_edge_scale(const EqfHeadLayout* lay, const float* alpha, const float* const* G,
                                   const int64_t* dst, int64_t n_edges, float* const* out, void* stream) {
  HeadArgs a;
  int rc = fill_head_args(lay, a);
  if (rc != EQF_OK || n_edges == 0) return rc;
  if (G == nullptr || dst == nullptr || out == nullptr) { set_error("eqf_attn_edge_scale: null pointer"); return EQF_ERR_INVALID; }
  int max_rowlen = 0;
  for (int g = 0; g < a.n_groups; ++g) {
    if (G[g] == nullptr || out[g] == nullptr) { set_error("eqf_attn_edge_scale: null group"); return EQF_ERR_INVALID; }
    a.G[g] = G[g]; a.out[g] = out[g];
    if (a.rowlen[g] > max_rowlen) max_rowlen = a.rowlen[g];
  }
  if (vec_ok(a)) {
    long long vb = (n_edges + 7) / 8;
    if (vb > 132LL * 16) vb = 132LL * 16;
    edge_scale_vec_kernel<<<(unsigned)(vb < 1 ? 1 : vb), 256, 0, (cudaStream_t)stream>>>(
        a, alpha, reinterpret_cast<const long long*>(dst), n_edges);
    return check_cuda(cudaGetLastError(), "edge_scale_vec_kernel launch");
  }
  long long blocks = (n_edges * max_rowlen + 255) / 256;
  if (blocks > 132LL * 32) blocks = 132LL * 32;
  if (blocks < 1) blocks = 1;
  dim3 grid((unsigned)blocks, (unsigned)a.n_groups);
  edge_scale_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, alpha, reinterpret_cast<const long long*>(dst), n_edges);
  return check_cuda(cudaGetLastError(), "edge_scale_kernel launch");
}
