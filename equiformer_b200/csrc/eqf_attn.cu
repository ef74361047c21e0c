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

#include <type_traits>

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
// (the eager version is a multiply, an index_add into [N, H], a gather back to [E, H], a multiply and a subtract).
// `keep` (optional, [E, H]): the attention-dropout mask applied after the softmax; the cotangent is then ga * keep.
__global__ void __launch_bounds__(256) seg_softmax_bwd_kernel(const float* __restrict__ alpha, const float* __restrict__ ga,
                                                              const float* __restrict__ keep,
                                                              const long long* __restrict__ row_ptr, long long n_nodes, int H,
                                                              float* __restrict__ gz) {
  const long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= n_nodes) return;
  const int lane = threadIdx.x & 31;
  const long long r0 = row_ptr[t], r1 = row_ptr[t + 1];
  for (int h = 0; h < H; ++h) {
    float s = 0.f;
    for (long long e = r0 + lane; e < r1; e += 32) {
      const float g = keep ? __ldg(ga + e * H + h) * __ldg(keep + e * H + h) : __ldg(ga + e * H + h);
      s += __ldg(alpha + e * H + h) * g;
    }
    s = warp_add(s);
    for (long long e = r0 + lane; e < r1; e += 32) {
      const float a = __ldg(alpha + e * H + h);
      const float g = keep ? __ldg(ga + e * H + h) * __ldg(keep + e * H + h) : __ldg(ga + e * H + h);
      gz[e * H + h] = a * (g - s);
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

// elementwise: out[g][e,j] = alpha[e,head(j)] (* keep[e,head(j)]) * G[g][dst[e],j]; grid.y = group
__global__ void __launch_bounds__(256) edge_scale_kernel(HeadArgs a, const float* __restrict__ alpha,
                                                         const float* __restrict__ keep,
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
    if (alpha != nullptr) {
      const long long k = e * H + (j % C) / ch;
      v *= keep ? __ldg(alpha + k) * __ldg(keep + k) : __ldg(alpha + k);
    }
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
// that own the first channel of each head in the 0e group) because the backward needs it.  `keep` (optional, [E, H]) is
// the attention-dropout mask (0 or 1/(1-p)): the sum then runs over alpha_e keep_e V_e, while alpha stays unmasked.
__global__ void __launch_bounds__(256) softmax_aggregate_vec_kernel(HeadArgs a, const float* __restrict__ z,
                                                                    const float* __restrict__ keep,
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
    float a0 = expf(__ldg(z + e * H + h) - m) * inv, a1 = expf(__ldg(z + (e + 1) * H + h) - m) * inv;
    const float4 v0 = ldv(v + e * rowlen), v1 = ldv(v + (e + 1) * rowlen);
    if (writer) { alpha_out[e * H + h] = a0; alpha_out[(e + 1) * H + h] = a1; }
    if (keep) { a0 *= __ldg(keep + e * H + h); a1 *= __ldg(keep + (e + 1) * H + h); }
    acc0.x = fmaf(a0, v0.x, acc0.x); acc0.y = fmaf(a0, v0.y, acc0.y); acc0.z = fmaf(a0, v0.z, acc0.z); acc0.w = fmaf(a0, v0.w, acc0.w);
    acc1.x = fmaf(a1, v1.x, acc1.x); acc1.y = fmaf(a1, v1.y, acc1.y); acc1.z = fmaf(a1, v1.z, acc1.z); acc1.w = fmaf(a1, v1.w, acc1.w);
  }
  if (e < r1) {
    float a0 = expf(__ldg(z + e * H + h) - m) * inv;
    const float4 v0 = ldv(v + e * rowlen);
    if (writer) alpha_out[e * H + h] = a0;
    if (keep) a0 *= __ldg(keep + e * H + h);
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

// one warp per edge: out[g][e, j] = alpha[e, head(j)] (* keep[e, head(j)]) * G[g][dst[e], j]
__global__ void __launch_bounds__(256) edge_scale_vec_kernel(HeadArgs a, const float* __restrict__ alpha,
                                                             const float* __restrict__ keep,
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
          const long long k = e * a.n_heads + (j % C) / ch;
          const float s = keep ? __ldg(alpha + k) * __ldg(keep + k) : __ldg(alpha + k);
          v.x *= s; v.y *= s; v.z *= s; v.w *= s;
        }
        *reinterpret_cast<float4*>(o + j) = v;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ dot-product attention
// The DP layer's q[dst] . k -> segment softmax -> (dropout) -> sum alpha v (ref nets/dp_attention_transformer.py:145-151)
// in one launch, reading keys and values straight from the key / value blocks kv[g] = [E, d_g, 2 C_g] (keys in channels
// [0, C_g), values in [C_g, 2 C_g)).  One warp per destination node, grid-stride over the nodes; a lane owns up to S float4
// slots of the node row (all groups concatenated, slot = lane + 32 s), every slot inside one head.  Two passes over the
// segment: the first reads the keys, forms z per head (a warp reduction per head), keeps an online max and sum of
// exponentials and parks z in alpha[e, h]; the second turns z into alpha = exp(z - max) / (sum + 1e-16) over it and
// accumulates alpha keep v from the values.  Lane h writes and re-reads its own alpha[e, h], so no cross-lane ordering is
// needed; a segment of any length costs no shared memory.  The key / value row is read once in all, the q row once per
// node; no atomics, and the order of every sum is fixed.
struct DotArgs {
  int n_groups, n_slots;
  int C[EQF_MAX_BLOCKS];                 // channels of group g in q / out (kv rows hold 2 C)
  int d[EQF_MAX_BLOCKS];
  int slot_start[EQF_MAX_BLOCKS + 1];    // prefix sum of d C / 4
  const float* q[EQF_MAX_BLOCKS];        // [N, d, C]
  const float* kv[EQF_MAX_BLOCKS];       // [E, d, 2C]
  const float* G[EQF_MAX_BLOCKS];        // [N, d, C]  (backward: d L / d out)
  float* out[EQF_MAX_BLOCKS];            // [N, d, C]  forward: out; backward: gq
  float* gkv[EQF_MAX_BLOCKS];            // [E, d, 2C] (backward)
};

constexpr int DOT_MAX_SLOTS = 8;         // float4 slots per lane: node rows of up to 1024 floats

__device__ __forceinline__ float dot4(float4 x, float4 y) { return x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w; }
__device__ __forceinline__ void fma4(float4& acc, float s, float4 v) {
  acc.x = fmaf(s, v.x, acc.x); acc.y = fmaf(s, v.y, acc.y); acc.z = fmaf(s, v.z, acc.z); acc.w = fmaf(s, v.w, acc.w);
}
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// slot c of a group-concatenated node row: its group, offset in the node row, offset in the kv row, head
__device__ __forceinline__ void dot_slot(const DotArgs& a, int H, int c, int& g, int& node_off, int& kv_off, int& head) {
  g = 0;
  while (g + 1 < a.n_groups && c >= a.slot_start[g + 1]) ++g;
  const int C = a.C[g], local = (c - a.slot_start[g]) * 4;
  const int i = local / C, j = local - i * C;
  node_off = local; kv_off = i * 2 * C + j; head = j / (C / H);
}

// the lane's slots, fixed for the whole kernel: head (-1: no slot), kv row stride, value offset C and the key columns of
// kv / gkv at edge 0 (the value columns are C further)
template <int H, int S>
struct DotSlots {
  int head[S], stride[S], C[S];
  const float* k[S];
  float* gk[S];
  __device__ __forceinline__ DotSlots(const DotArgs& a, int lane) {
#pragma unroll
    for (int s = 0; s < S; ++s) {
      const int c = lane + 32 * s;
      int g, node_off, kv_off, h;
      dot_slot(a, H, c < a.n_slots ? c : 0, g, node_off, kv_off, h);
      head[s] = c < a.n_slots ? h : -1;
      stride[s] = 2 * a.C[g] * a.d[g];
      C[s] = a.C[g];
      k[s] = a.kv[g] + kv_off;
      gk[s] = a.gkv[g] == nullptr ? nullptr : a.gkv[g] + kv_off;
    }
  }
};

// element offset of slot c in node row t, and its group
__device__ __forceinline__ long long node_index(const DotArgs& a, int H, int c, long long t, int& g) {
  int node_off, kv_off, h;
  dot_slot(a, H, c, g, node_off, kv_off, h);
  return t * (long long)(a.d[g] * a.C[g]) + node_off;
}

template <int H, int S>
__device__ __forceinline__ void load_node_row(const DotArgs& a, const float* const* base, const DotSlots<H, S>& sl, int lane,
                                              long long t, float4 (&x)[S]) {
#pragma unroll
  for (int s = 0; s < S; ++s) {
    x[s] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (sl.head[s] >= 0) {
      int g;
      const long long i = node_index(a, H, lane + 32 * s, t, g);
      x[s] = ldv(base[g] + i);
    }
  }
}

template <int H, int S>
__device__ __forceinline__ void store_node_row(const DotArgs& a, const DotSlots<H, S>& sl, int lane, long long t,
                                               const float4 (&x)[S]) {
#pragma unroll
  for (int s = 0; s < S; ++s) {
    if (sl.head[s] >= 0) {
      int g;
      const long long i = node_index(a, H, lane + 32 * s, t, g);
      st4(a.out[g] + i, x[s]);
    }
  }
}

// per-head sums of the lanes' slot products: every lane gets all H
template <int H, int S>
__device__ __forceinline__ void head_sums(const float (&p)[S], const int (&head)[S], float (&z)[H]) {
#pragma unroll
  for (int h = 0; h < H; ++h) {
    float acc = 0.f;
#pragma unroll
    for (int s = 0; s < S; ++s) acc += (head[s] == h) ? p[s] : 0.f;
    z[h] = warp_add(acc);
  }
}

template <int H>
__device__ __forceinline__ float lane_pick(const float (&x)[H], int lane) {
  float r = 0.f;
#pragma unroll
  for (int h = 0; h < H; ++h) r = (lane == h) ? x[h] : r;
  return r;
}

template <int H, int S>
__global__ void __launch_bounds__(256) dot_softmax_aggregate_kernel(DotArgs a, const float* __restrict__ keep,
                                                                    const long long* __restrict__ row_ptr, long long n_nodes,
                                                                    float* __restrict__ alpha) {
  const int lane = threadIdx.x & 31;
  const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
  const DotSlots<H, S> sl(a, lane);
  for (long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < n_nodes; t += n_warps) {
    const long long r0 = row_ptr[t], r1 = row_ptr[t + 1];
    float4 q[S];
    load_node_row<H, S>(a, a.q, sl, lane, t, q);
    // pass 1 (keys): z per head, online max and sum of exponentials; z parked in alpha
    float m[H], sum[H];
#pragma unroll
    for (int h = 0; h < H; ++h) { m[h] = -CUDART_INF_F; sum[h] = 0.f; }
    for (long long e = r0; e < r1; ++e) {
      float p[S];
#pragma unroll
      for (int s = 0; s < S; ++s) p[s] = sl.head[s] >= 0 ? dot4(q[s], ldv(sl.k[s] + e * sl.stride[s])) : 0.f;
      float z[H];
      head_sums<H, S>(p, sl.head, z);
#pragma unroll
      for (int h = 0; h < H; ++h) {
        if (z[h] > m[h]) { sum[h] = sum[h] * expf(m[h] - z[h]) + 1.f; m[h] = z[h]; }
        else sum[h] += expf(z[h] - m[h]);
      }
      if (lane < H) alpha[e * H + lane] = lane_pick<H>(z, lane);
    }
    // pass 2 (values): alpha over z, out = sum alpha keep v
    float my_m = 0.f, my_inv = 0.f;
#pragma unroll
    for (int h = 0; h < H; ++h) {
      if (lane == h) { my_m = m[h]; my_inv = 1.f / (sum[h] + 1e-16f); }
    }
    float4 acc[S];
#pragma unroll
    for (int s = 0; s < S; ++s) acc[s] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long e = r0; e < r1; ++e) {
      float w = 0.f;
      if (lane < H) {
        const float al = expf(alpha[e * H + lane] - my_m) * my_inv;
        alpha[e * H + lane] = al;
        w = keep ? al * __ldg(keep + e * H + lane) : al;
      }
#pragma unroll
      for (int s = 0; s < S; ++s) {
        const float ws = __shfl_sync(0xffffffffu, w, sl.head[s] & 31);
        if (sl.head[s] >= 0) fma4(acc[s], ws, ldv(sl.k[s] + e * sl.stride[s] + sl.C[s]));
      }
    }
    store_node_row<H, S>(a, sl, lane, t, acc);
  }
}

// Backward of the kernel above, same warp-per-node layout; G = d L / d out.  Pass 1 (values): ga_e = v_e . G[t] per head
// (parked in work[e, h] by lane h), s_t = sum alpha keep ga and gv_e = alpha_e keep_e G[t].  Pass 2 (keys):
// gz_e = alpha_e (keep_e ga_e - s_t), gk_e = gz_e q[t] and gq[t] = sum gz_e k_e.  Every output row has one owner; the key /
// value row is read once and its gradient row written once.
template <int H, int S>
__global__ void __launch_bounds__(256) dot_softmax_aggregate_bwd_kernel(DotArgs a, const float* __restrict__ alpha,
                                                                        const float* __restrict__ keep,
                                                                        const long long* __restrict__ row_ptr,
                                                                        long long n_nodes, float* __restrict__ work) {
  const int lane = threadIdx.x & 31;
  const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
  const DotSlots<H, S> sl(a, lane);
  for (long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < n_nodes; t += n_warps) {
    const long long r0 = row_ptr[t], r1 = row_ptr[t + 1];
    float4 x[S];
    load_node_row<H, S>(a, a.G, sl, lane, t, x);
    float s_t = 0.f;                   // lane h: sum over the segment of alpha keep ga for head h
    for (long long e = r0; e < r1; ++e) {
      float p[S];
#pragma unroll
      for (int s = 0; s < S; ++s)
        p[s] = sl.head[s] >= 0 ? dot4(x[s], ldv(sl.k[s] + e * sl.stride[s] + sl.C[s])) : 0.f;
      float ga[H];
      head_sums<H, S>(p, sl.head, ga);
      float w = 0.f;
      if (lane < H) {
        const float g = lane_pick<H>(ga, lane);
        w = __ldg(alpha + e * H + lane);
        if (keep) w *= __ldg(keep + e * H + lane);
        s_t = fmaf(w, g, s_t);
        work[e * H + lane] = g;
      }
#pragma unroll
      for (int s = 0; s < S; ++s) {
        const float ws = __shfl_sync(0xffffffffu, w, sl.head[s] & 31);
        if (sl.head[s] >= 0)
          st4(sl.gk[s] + e * sl.stride[s] + sl.C[s], make_float4(ws * x[s].x, ws * x[s].y, ws * x[s].z, ws * x[s].w));
      }
    }
    load_node_row<H, S>(a, a.q, sl, lane, t, x);
    float4 gq[S];
#pragma unroll
    for (int s = 0; s < S; ++s) gq[s] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long e = r0; e < r1; ++e) {
      float gz = 0.f;
      if (lane < H) {
        const float kp = keep ? __ldg(keep + e * H + lane) : 1.f;
        gz = __ldg(alpha + e * H + lane) * (kp * work[e * H + lane] - s_t);
      }
#pragma unroll
      for (int s = 0; s < S; ++s) {
        const float gs = __shfl_sync(0xffffffffu, gz, sl.head[s] & 31);
        if (sl.head[s] >= 0) {
          fma4(gq[s], gs, ldv(sl.k[s] + e * sl.stride[s]));
          st4(sl.gk[s] + e * sl.stride[s], make_float4(gs * x[s].x, gs * x[s].y, gs * x[s].z, gs * x[s].w));
        }
      }
    }
    store_node_row<H, S>(a, sl, lane, t, gq);
  }
}

// ------------------------------------------------------------------------------------------------ linear-message attention
// The linear-message GraphAttention (ref nets/graph_attention_transformer.py:497-513 with nonlinear_message=False) from the
// output of sep.lin on: z = sum_k c SLR(t0[alpha k]) alpha_dot[k] per head, the segment softmax, (dropout) and the weighted
// sum of the value scalars and the l >= 1 value blocks, in one launch.  The 0e row t0 [E, H (A + R)] is read in place: head
// h owns the alpha pre-activations [h (A + R), h (A + R) + A) and the value scalars [h (A + R) + A, (h + 1)(A + R)) (the
// Vec2AttnHeads split).  Same warp-per-node scheme as the dot-product kernel: a lane owns up to SA float4 slots of the
// alpha row and up to SV float4 slots of the value row (value groups concatenated: g = 0 the value scalars inside t0,
// g >= 1 the blocks V[g] = [E, d_g, H C_g]), every slot inside one head.  Pass 1 reads the alpha channels, forms z per
// head and keeps an online max and sum of exponentials, parking z in alpha[e, h]; pass 2 turns it into alpha and
// accumulates alpha keep v.  Lane h alone writes and re-reads alpha[e, h]; no atomics, fixed summation order.
struct MlpArgs {
  int H, A, R, T;                        // heads; alpha / value-scalar channels per head; t0 row length H (A + R)
  int n_groups, n_aslots, n_vslots;      // value groups (g = 0: the value scalars); float4 slots of alpha / value rows
  int d[EQF_MAX_BLOCKS];                 // components of value group g (d[0] = 1)
  int C[EQF_MAX_BLOCKS];                 // channels per head of value group g (C[0] = R)
  int vslot_start[EQF_MAX_BLOCKS + 1];   // prefix sum of d H C / 4
  float c_slr, k1, k2;                   // alpha_act: c ((1+a)/2 x + (1-a)/2 x (2 sigmoid(x) - 1))
  const float* t0;                       // [E, T]
  const float* V[EQF_MAX_BLOCKS];        // g >= 1: [E, d, H C]
  const float* alpha_dot;                // [H, A]
  const float* G[EQF_MAX_BLOCKS];        // backward: d L / d out, [N, d, H C]
  float* out[EQF_MAX_BLOCKS];            // forward: [N, d, H C]
  float* gt0;                            // backward: [E, T], every channel written
  float* gV[EQF_MAX_BLOCKS];             // backward, g >= 1: [E, d, H C]
  float* gdot_part;                      // backward: per-CTA partial sums of d L / d alpha_dot, [grid, H A]
};

__device__ __forceinline__ float slr_sig(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float mlp_act(const MlpArgs& a, float x) {
  return a.c_slr * (a.k1 * x + a.k2 * x * (2.f * slr_sig(x) - 1.f));
}
__device__ __forceinline__ float mlp_dact(const MlpArgs& a, float x) {
  const float s = slr_sig(x);
  return a.c_slr * (a.k1 + a.k2 * ((2.f * s - 1.f) + 2.f * x * s * (1.f - s)));
}

// the lane's slots, fixed for the whole kernel.  Alpha slot c (float4 c of alpha_dot): head c / (A / 4), t0 column
// head (A + R) + 4 (c % (A / 4)).  Value slot c: group g, offset `local` in the group's node row; its edge row is t0
// (g = 0, column head (A + R) + A + local % R) or V[g] (column local).  `node` is the node-row buffer (out in the
// forward, G in the backward), `grad` the edge-row gradient (backward only).
template <int SA, int SV>
struct MlpSlots {
  int ahead[SA], aoff[SA];
  float4 ad[SA];
  int vhead[SV], vstride[SV], nrow[SV];
  const float* v[SV];
  float* gv[SV];
  float* node[SV];
  __device__ __forceinline__ MlpSlots(const MlpArgs& a, int lane, float* const* node_rows, bool backward) {
    const int H4 = a.A / 4;
#pragma unroll
    for (int s = 0; s < SA; ++s) {
      const int c = lane + 32 * s;
      const bool on = c < a.n_aslots;
      const int h = (on ? c : 0) / H4;
      ahead[s] = on ? h : -1;
      aoff[s] = h * (a.A + a.R) + 4 * ((on ? c : 0) % H4);
      ad[s] = on ? ldv(a.alpha_dot + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int s = 0; s < SV; ++s) {
      const int c0 = lane + 32 * s;
      const bool on = c0 < a.n_vslots;
      const int c = on ? c0 : 0;
      int g = 0;
      while (g + 1 < a.n_groups && c >= a.vslot_start[g + 1]) ++g;
      const int HC = a.C[g] * a.H;
      const int local = (c - a.vslot_start[g]) * 4;
      const int j = local % HC, h = j / a.C[g];
      vhead[s] = on ? h : -1;
      nrow[s] = a.d[g] * HC;
      node[s] = node_rows[g] + local;
      if (g == 0) {
        const int col = h * (a.A + a.R) + a.A + (j - h * a.C[0]);
        vstride[s] = a.T;
        v[s] = a.t0 + col;
        gv[s] = backward ? a.gt0 + col : nullptr;
      } else {
        vstride[s] = nrow[s];
        v[s] = a.V[g] + local;
        gv[s] = backward ? a.gV[g] + local : nullptr;
      }
    }
  }
};

template <int H, int SA, int SV>
__global__ void __launch_bounds__(256) mlp_softmax_aggregate_kernel(MlpArgs a, const float* __restrict__ keep,
                                                                    const long long* __restrict__ row_ptr, long long n_nodes,
                                                                    float* __restrict__ alpha) {
  const int lane = threadIdx.x & 31;
  const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
  const MlpSlots<SA, SV> sl(a, lane, a.out, false);
  for (long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < n_nodes; t += n_warps) {
    const long long r0 = row_ptr[t], r1 = row_ptr[t + 1];
    // pass 1 (alpha channels): z per head; lane h keeps head h's online max and sum of exponentials, z parked in alpha
    float m = -CUDART_INF_F, sum = 0.f;
    for (long long e = r0; e < r1; ++e) {
      const float* row = a.t0 + e * a.T;
      float p[SA];
#pragma unroll
      for (int s = 0; s < SA; ++s) {
        p[s] = 0.f;
        if (sl.ahead[s] >= 0) {
          const float4 x = ldv(row + sl.aoff[s]);
          p[s] = mlp_act(a, x.x) * sl.ad[s].x + mlp_act(a, x.y) * sl.ad[s].y + mlp_act(a, x.z) * sl.ad[s].z +
                 mlp_act(a, x.w) * sl.ad[s].w;
        }
      }
      float z[H];
      head_sums<H, SA>(p, sl.ahead, z);
      if (lane < H) {
        const float zl = lane_pick<H>(z, lane);
        if (zl > m) { sum = sum * expf(m - zl) + 1.f; m = zl; }
        else sum += expf(zl - m);
        alpha[e * H + lane] = zl;
      }
    }
    // pass 2 (values): alpha over z, out = sum alpha keep v
    const float inv = 1.f / (sum + 1e-16f);
    float4 acc[SV];
#pragma unroll
    for (int s = 0; s < SV; ++s) acc[s] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long e = r0; e < r1; ++e) {
      float w = 0.f;
      if (lane < H) {
        const float al = expf(alpha[e * H + lane] - m) * inv;
        alpha[e * H + lane] = al;
        w = keep ? al * __ldg(keep + e * H + lane) : al;
      }
#pragma unroll
      for (int s = 0; s < SV; ++s) {
        const float ws = __shfl_sync(0xffffffffu, w, sl.vhead[s] & 31);
        if (sl.vhead[s] >= 0) fma4(acc[s], ws, ldv(sl.v[s] + e * sl.vstride[s]));
      }
    }
#pragma unroll
    for (int s = 0; s < SV; ++s)
      if (sl.vhead[s] >= 0) st4(sl.node[s] + t * sl.nrow[s], acc[s]);
  }
}

// Backward of the kernel above, same layout; G = d L / d out.  Pass 1 (values): ga_e = v_e . G[t] per head (parked in
// work[e, h] by lane h), s_t = sum alpha keep ga and gv_e = alpha_e keep_e G[t] (the value channels of gt0 and gV).
// Pass 2 (alpha channels): gz_e = alpha_e (keep_e ga_e - s_t), gt0 = gz alpha_dot act'(t0) and the lane's share of
// d L / d alpha_dot = sum_e gz act(t0) in registers.  At the end the CTA adds its warps' shares in warp order (shared
// memory, no atomics) into gdot_part[blockIdx.x]; eqf_colsum reduces the rows.  Every output element has one owner.
template <int H, int SA, int SV>
__global__ void __launch_bounds__(256) mlp_softmax_aggregate_bwd_kernel(MlpArgs a, const float* __restrict__ alpha,
                                                                        const float* __restrict__ keep,
                                                                        const long long* __restrict__ row_ptr,
                                                                        long long n_nodes, float* __restrict__ work) {
  __shared__ float4 red[8][SA * 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
  const MlpSlots<SA, SV> sl(a, lane, const_cast<float* const*>(a.G), true);
  float4 gdot[SA];
#pragma unroll
  for (int s = 0; s < SA; ++s) gdot[s] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long t = (long long)blockIdx.x * (blockDim.x >> 5) + warp; t < n_nodes; t += n_warps) {
    const long long r0 = row_ptr[t], r1 = row_ptr[t + 1];
    float4 x[SV];
#pragma unroll
    for (int s = 0; s < SV; ++s) x[s] = sl.vhead[s] >= 0 ? ldv(sl.node[s] + t * sl.nrow[s]) : make_float4(0.f, 0.f, 0.f, 0.f);
    float s_t = 0.f;                   // lane h: sum over the segment of alpha keep ga for head h
    for (long long e = r0; e < r1; ++e) {
      float p[SV];
#pragma unroll
      for (int s = 0; s < SV; ++s) p[s] = sl.vhead[s] >= 0 ? dot4(x[s], ldv(sl.v[s] + e * sl.vstride[s])) : 0.f;
      float ga[H];
      head_sums<H, SV>(p, sl.vhead, ga);
      float w = 0.f;
      if (lane < H) {
        const float g = lane_pick<H>(ga, lane);
        w = __ldg(alpha + e * H + lane);
        if (keep) w *= __ldg(keep + e * H + lane);
        s_t = fmaf(w, g, s_t);
        work[e * H + lane] = g;
      }
#pragma unroll
      for (int s = 0; s < SV; ++s) {
        const float ws = __shfl_sync(0xffffffffu, w, sl.vhead[s] & 31);
        if (sl.vhead[s] >= 0)
          st4(sl.gv[s] + e * sl.vstride[s], make_float4(ws * x[s].x, ws * x[s].y, ws * x[s].z, ws * x[s].w));
      }
    }
    for (long long e = r0; e < r1; ++e) {
      float gz = 0.f;
      if (lane < H) {
        const float kp = keep ? __ldg(keep + e * H + lane) : 1.f;
        gz = __ldg(alpha + e * H + lane) * (kp * work[e * H + lane] - s_t);
      }
#pragma unroll
      for (int s = 0; s < SA; ++s) {
        const float gs = __shfl_sync(0xffffffffu, gz, sl.ahead[s] & 31);
        if (sl.ahead[s] >= 0) {
          const float4 xa = ldv(a.t0 + e * a.T + sl.aoff[s]);
          const float4 ad = sl.ad[s];
          st4(a.gt0 + e * a.T + sl.aoff[s], make_float4(gs * ad.x * mlp_dact(a, xa.x), gs * ad.y * mlp_dact(a, xa.y),
                                                         gs * ad.z * mlp_dact(a, xa.z), gs * ad.w * mlp_dact(a, xa.w)));
          fma4(gdot[s], gs, make_float4(mlp_act(a, xa.x), mlp_act(a, xa.y), mlp_act(a, xa.z), mlp_act(a, xa.w)));
        }
      }
    }
  }
#pragma unroll
  for (int s = 0; s < SA; ++s) red[warp][s * 32 + lane] = gdot[s];
  __syncthreads();
  for (int c = threadIdx.x; c < a.n_aslots; c += blockDim.x) {
    float4 r = red[0][c];
#pragma unroll
    for (int w = 1; w < 8; ++w) {
      const float4 q = red[w][c];
      r.x += q.x; r.y += q.y; r.z += q.z; r.w += q.w;
    }
    st4(a.gdot_part + (long long)blockIdx.x * 4 * a.n_aslots + 4 * c, r);
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

extern "C" int eqf_seg_softmax_bwd(const float* alpha, const float* ga, const float* keep, const int64_t* row_ptr,
                                   int64_t n_nodes, int32_t n_heads, float* gz, void* stream) {
  if (n_nodes == 0) return EQF_OK;
  if (!alpha || !ga || !row_ptr || !gz || n_heads < 1) { set_error("eqf_seg_softmax_bwd: bad arguments"); return EQF_ERR_INVALID; }
  const int wpb = 8;
  const long long blocks = (n_nodes + wpb - 1) / wpb;
  seg_softmax_bwd_kernel<<<(unsigned)blocks, wpb * 32, 0, (cudaStream_t)stream>>>(
      alpha, ga, keep, reinterpret_cast<const long long*>(row_ptr), n_nodes, n_heads, gz);
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
extern "C" int eqf_attn_softmax_aggregate(const EqfHeadLayout* lay, const float* z, const float* keep, const float* const* V,
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
      a, z, keep, reinterpret_cast<const long long*>(row_ptr), n_nodes, alpha);
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

extern "C" int eqf_attn_edge_scale(const EqfHeadLayout* lay, const float* alpha, const float* keep, const float* const* G,
                                   const int64_t* dst, int64_t n_edges, float* const* out, void* stream) {
  HeadArgs a;
  int rc = fill_head_args(lay, a);
  if (rc != EQF_OK || n_edges == 0) return rc;
  if (G == nullptr || dst == nullptr || out == nullptr) { set_error("eqf_attn_edge_scale: null pointer"); return EQF_ERR_INVALID; }
  if (keep != nullptr && alpha == nullptr) { set_error("eqf_attn_edge_scale: keep needs alpha"); return EQF_ERR_INVALID; }
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
        a, alpha, keep, reinterpret_cast<const long long*>(dst), n_edges);
    return check_cuda(cudaGetLastError(), "edge_scale_vec_kernel launch");
  }
  long long blocks = (n_edges * max_rowlen + 255) / 256;
  if (blocks > 132LL * 32) blocks = 132LL * 32;
  if (blocks < 1) blocks = 1;
  dim3 grid((unsigned)blocks, (unsigned)a.n_groups);
  edge_scale_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, alpha, keep, reinterpret_cast<const long long*>(dst), n_edges);
  return check_cuda(cudaGetLastError(), "edge_scale_kernel launch");
}

// ------------------------------------------------------------------------------------------------ dot-product attention
namespace {

// DotArgs from the q / out head layout; EQF_ERR_UNSUPPORTED outside the float4 layout (channels per head % 4), above
// DOT_MAX_SLOTS float4 slots per lane or for a head count without a kernel instance
int fill_dot_args(const EqfHeadLayout* lay, DotArgs& a, int& slots_per_lane, const char* what) {
  HeadArgs h;
  int rc = fill_head_args(lay, h);
  if (rc != EQF_OK) return rc;
  a.n_groups = h.n_groups;
  a.slot_start[0] = 0;
  for (int g = 0; g < EQF_MAX_BLOCKS; ++g) {
    a.q[g] = a.kv[g] = a.G[g] = nullptr; a.out[g] = a.gkv[g] = nullptr;
    a.C[g] = a.d[g] = 0;
  }
  const int H = h.n_heads;
  bool ok = H == 1 || H == 2 || H == 4 || H == 8 || H == 16;
  for (int g = 0; g < h.n_groups; ++g) {
    a.C[g] = h.C[g]; a.d[g] = h.d[g];
    ok = ok && (h.C[g] / H) % 4 == 0;
    a.slot_start[g + 1] = a.slot_start[g] + h.d[g] * h.C[g] / 4;
  }
  a.n_slots = a.slot_start[a.n_groups];
  slots_per_lane = (a.n_slots + 31) / 32;
  if (!ok || slots_per_lane > DOT_MAX_SLOTS) {
    set_error(std::string(what) + ": layout not supported (channels per head must be a multiple of 4, at most 1024 "
              "channels per node row, 1 / 2 / 4 / 8 / 16 heads)");
    return EQF_ERR_UNSUPPORTED;
  }
  return EQF_OK;
}

// one warp per node, grid-stride: min(ceil(N / 8), 132 * 16) CTAs of 8 warps
unsigned dot_grid(long long n_nodes) {
  long long b = (n_nodes + 7) / 8;
  if (b > 132LL * 16) b = 132LL * 16;
  return (unsigned)(b < 1 ? 1 : b);
}

template <int S, typename Launch>
int dispatch_heads(int H, Launch&& launch) {
  switch (H) {
    case 1: launch(std::integral_constant<int, 1>{}, std::integral_constant<int, S>{}); break;
    case 2: launch(std::integral_constant<int, 2>{}, std::integral_constant<int, S>{}); break;
    case 4: launch(std::integral_constant<int, 4>{}, std::integral_constant<int, S>{}); break;
    case 8: launch(std::integral_constant<int, 8>{}, std::integral_constant<int, S>{}); break;
    default: launch(std::integral_constant<int, 16>{}, std::integral_constant<int, S>{}); break;
  }
  return EQF_OK;
}

// float4 slots per lane: 4 (node rows up to 512 floats: the QM9 L2 heads), 5 (640: OC20 L1) or 8 (1024: MD17 L3); the
// register count grows with S, so the shipped layouts get the smallest instance that holds their row
template <typename Launch>
void dispatch_dot(int H, int slots_per_lane, Launch&& launch) {
  if (slots_per_lane <= 4) dispatch_heads<4>(H, launch);
  else if (slots_per_lane == 5) dispatch_heads<5>(H, launch);
  else dispatch_heads<DOT_MAX_SLOTS>(H, launch);
}

}  // namespace

extern "C" int eqf_attn_dot_softmax_aggregate(const EqfHeadLayout* lay, const float* const* q, const float* const* kv,
                                              const float* keep, const int64_t* row_ptr, int64_t n_nodes, float* const* out,
                                              float* alpha, void* stream) {
  DotArgs a;
  int S = 0;
  int rc = fill_dot_args(lay, a, S, "eqf_attn_dot_softmax_aggregate");
  if (rc != EQF_OK || n_nodes == 0) return rc;
  if (q == nullptr || kv == nullptr || out == nullptr || row_ptr == nullptr || alpha == nullptr) {
    set_error("eqf_attn_dot_softmax_aggregate: null pointer"); return EQF_ERR_INVALID;
  }
  for (int g = 0; g < a.n_groups; ++g) {
    if (q[g] == nullptr || kv[g] == nullptr || out[g] == nullptr) {
      set_error("eqf_attn_dot_softmax_aggregate: null group"); return EQF_ERR_INVALID;
    }
    a.q[g] = q[g]; a.kv[g] = kv[g]; a.out[g] = out[g];
  }
  const long long* rp = reinterpret_cast<const long long*>(row_ptr);
  cudaStream_t st = (cudaStream_t)stream;
  dispatch_dot(lay->n_heads, S, [&](auto Hc, auto Sc) {
    dot_softmax_aggregate_kernel<decltype(Hc)::value, decltype(Sc)::value><<<dot_grid(n_nodes), 256, 0, st>>>(
        a, keep, rp, n_nodes, alpha);
  });
  return check_cuda(cudaGetLastError(), "dot_softmax_aggregate_kernel launch");
}

extern "C" int eqf_attn_dot_softmax_aggregate_bwd(const EqfHeadLayout* lay, const float* const* G, const float* const* q,
                                                  const float* const* kv, const float* alpha, const float* keep,
                                                  const int64_t* row_ptr, int64_t n_nodes, float* const* gq,
                                                  float* const* gkv, float* work, void* stream) {
  DotArgs a;
  int S = 0;
  int rc = fill_dot_args(lay, a, S, "eqf_attn_dot_softmax_aggregate_bwd");
  if (rc != EQF_OK || n_nodes == 0) return rc;
  if (G == nullptr || q == nullptr || kv == nullptr || alpha == nullptr || row_ptr == nullptr || gq == nullptr ||
      gkv == nullptr || work == nullptr) {
    set_error("eqf_attn_dot_softmax_aggregate_bwd: null pointer"); return EQF_ERR_INVALID;
  }
  for (int g = 0; g < a.n_groups; ++g) {
    if (G[g] == nullptr || q[g] == nullptr || kv[g] == nullptr || gq[g] == nullptr || gkv[g] == nullptr) {
      set_error("eqf_attn_dot_softmax_aggregate_bwd: null group"); return EQF_ERR_INVALID;
    }
    a.G[g] = G[g]; a.q[g] = q[g]; a.kv[g] = kv[g]; a.out[g] = gq[g]; a.gkv[g] = gkv[g];
  }
  const long long* rp = reinterpret_cast<const long long*>(row_ptr);
  cudaStream_t st = (cudaStream_t)stream;
  dispatch_dot(lay->n_heads, S, [&](auto Hc, auto Sc) {
    dot_softmax_aggregate_bwd_kernel<decltype(Hc)::value, decltype(Sc)::value><<<dot_grid(n_nodes), 256, 0, st>>>(
        a, alpha, keep, rp, n_nodes, work);
  });
  return check_cuda(cudaGetLastError(), "dot_softmax_aggregate_bwd_kernel launch");
}

// ------------------------------------------------------------------------------------------------ linear-message attention
namespace {

// float4 slots per lane of the kernel instance for H heads: <SA 2, SV 5> for 8 heads (alpha rows of up to 256 floats,
// value rows of up to 640: OC20 L1), <SA 1, SV 4> for 2 and 4 (128 / 512: the QM9 / MD17 L2 heads)
int mlp_alpha_slots(int H) { return H == 8 ? 2 : 1; }
int mlp_value_slots(int H) { return H == 8 ? 5 : 4; }

// MlpArgs from the output layout `lay` (group 0: the value scalars [N, 1, H R]; groups >= 1: the l >= 1 blocks) and the
// alpha channels per head; EQF_ERR_UNSUPPORTED outside the float4 layout (A, R and every C_g per head % 4), above the
// slot counts of the instances or for a head count without one
int fill_mlp_args(const EqfHeadLayout* lay, int n_alpha, float c_slr, float slope, MlpArgs& a, const char* what) {
  HeadArgs h;
  int rc = fill_head_args(lay, h);
  if (rc != EQF_OK) return rc;
  const int H = h.n_heads;
  a.H = H; a.A = n_alpha; a.R = h.C[0] / H; a.T = H * (n_alpha + a.R);
  a.n_groups = h.n_groups;
  a.n_aslots = H * n_alpha / 4;
  a.vslot_start[0] = 0;
  a.c_slr = c_slr; a.k1 = 0.5f * (1.f + slope); a.k2 = 0.5f * (1.f - slope);
  a.t0 = a.alpha_dot = nullptr; a.gt0 = a.gdot_part = nullptr;
  bool ok = (H == 2 || H == 4 || H == 8) && n_alpha > 0 && n_alpha % 4 == 0 && h.d[0] == 1;
  for (int g = 0; g < EQF_MAX_BLOCKS; ++g) {
    a.V[g] = a.G[g] = nullptr; a.out[g] = a.gV[g] = nullptr;
    a.d[g] = a.C[g] = 0;
  }
  for (int g = 0; g < h.n_groups; ++g) {
    a.d[g] = h.d[g]; a.C[g] = h.C[g] / H;
    ok = ok && a.C[g] % 4 == 0;
    a.vslot_start[g + 1] = a.vslot_start[g] + h.d[g] * h.C[g] / 4;
  }
  a.n_vslots = a.vslot_start[a.n_groups];
  if (!ok || a.n_aslots > 32 * mlp_alpha_slots(H) || a.n_vslots > 32 * mlp_value_slots(H)) {
    set_error(std::string(what) + ": layout not supported (2 / 4 / 8 heads, a leading 0e value group, alpha and value "
              "channels per head multiples of 4, at most 128 alpha and 512 value channels per edge (256 and 640 with 8 "
              "heads))");
    return EQF_ERR_UNSUPPORTED;
  }
  return EQF_OK;
}

template <typename Launch>
void dispatch_mlp(int H, Launch&& launch) {
  switch (H) {
    case 2: launch(std::integral_constant<int, 2>{}, std::integral_constant<int, 1>{}, std::integral_constant<int, 4>{}); break;
    case 4: launch(std::integral_constant<int, 4>{}, std::integral_constant<int, 1>{}, std::integral_constant<int, 4>{}); break;
    default: launch(std::integral_constant<int, 8>{}, std::integral_constant<int, 2>{}, std::integral_constant<int, 5>{}); break;
  }
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

extern "C" int eqf_attn_mlp_rows(int64_t n_nodes) { return (int)dot_grid(n_nodes); }

extern "C" int eqf_attn_mlp_softmax_aggregate(const EqfHeadLayout* lay, int32_t n_alpha, float c_slr, float slope,
                                              const float* t0, const float* const* V, const float* alpha_dot,
                                              const float* keep, const int64_t* row_ptr, int64_t n_nodes,
                                              float* const* out, float* alpha, void* stream) {
  MlpArgs a;
  int rc = fill_mlp_args(lay, n_alpha, c_slr, slope, a, "eqf_attn_mlp_softmax_aggregate");
  if (rc != EQF_OK || n_nodes == 0) return rc;
  if (t0 == nullptr || alpha_dot == nullptr || row_ptr == nullptr || out == nullptr || alpha == nullptr ||
      (a.n_groups > 1 && V == nullptr)) {
    set_error("eqf_attn_mlp_softmax_aggregate: null pointer"); return EQF_ERR_INVALID;
  }
  a.t0 = t0; a.alpha_dot = alpha_dot;
  bool al = aligned16(t0) && aligned16(alpha_dot);
  for (int g = 0; g < a.n_groups; ++g) {
    if (out[g] == nullptr || (g > 0 && V[g - 1] == nullptr)) {
      set_error("eqf_attn_mlp_softmax_aggregate: null group"); return EQF_ERR_INVALID;
    }
    a.out[g] = out[g];
    if (g > 0) a.V[g] = V[g - 1];
    al = al && aligned16(a.out[g]) && (g == 0 || aligned16(a.V[g]));
  }
  if (!al) { set_error("eqf_attn_mlp_softmax_aggregate: operands must be 16-byte aligned"); return EQF_ERR_INVALID; }
  const long long* rp = reinterpret_cast<const long long*>(row_ptr);
  cudaStream_t st = (cudaStream_t)stream;
  dispatch_mlp(a.H, [&](auto Hc, auto SAc, auto SVc) {
    mlp_softmax_aggregate_kernel<decltype(Hc)::value, decltype(SAc)::value, decltype(SVc)::value>
        <<<dot_grid(n_nodes), 256, 0, st>>>(a, keep, rp, n_nodes, alpha);
  });
  return check_cuda(cudaGetLastError(), "mlp_softmax_aggregate_kernel launch");
}

extern "C" int eqf_attn_mlp_softmax_aggregate_bwd(const EqfHeadLayout* lay, int32_t n_alpha, float c_slr, float slope,
                                                  const float* const* G, const float* t0, const float* const* V,
                                                  const float* alpha_dot, const float* alpha, const float* keep,
                                                  const int64_t* row_ptr, int64_t n_nodes, float* gt0, float* const* gV,
                                                  float* work, float* gdot_part, void* stream) {
  MlpArgs a;
  int rc = fill_mlp_args(lay, n_alpha, c_slr, slope, a, "eqf_attn_mlp_softmax_aggregate_bwd");
  if (rc != EQF_OK || n_nodes == 0) return rc;
  if (G == nullptr || t0 == nullptr || alpha_dot == nullptr || alpha == nullptr || row_ptr == nullptr || gt0 == nullptr ||
      work == nullptr || gdot_part == nullptr || (a.n_groups > 1 && (V == nullptr || gV == nullptr))) {
    set_error("eqf_attn_mlp_softmax_aggregate_bwd: null pointer"); return EQF_ERR_INVALID;
  }
  a.t0 = t0; a.alpha_dot = alpha_dot; a.gt0 = gt0; a.gdot_part = gdot_part;
  bool al = aligned16(t0) && aligned16(alpha_dot) && aligned16(gt0) && aligned16(gdot_part);
  for (int g = 0; g < a.n_groups; ++g) {
    if (G[g] == nullptr || (g > 0 && (V[g - 1] == nullptr || gV[g - 1] == nullptr))) {
      set_error("eqf_attn_mlp_softmax_aggregate_bwd: null group"); return EQF_ERR_INVALID;
    }
    a.G[g] = G[g];
    if (g > 0) { a.V[g] = V[g - 1]; a.gV[g] = gV[g - 1]; }
    al = al && aligned16(a.G[g]) && (g == 0 || (aligned16(a.V[g]) && aligned16(a.gV[g])));
  }
  if (!al) { set_error("eqf_attn_mlp_softmax_aggregate_bwd: operands must be 16-byte aligned"); return EQF_ERR_INVALID; }
  const long long* rp = reinterpret_cast<const long long*>(row_ptr);
  cudaStream_t st = (cudaStream_t)stream;
  dispatch_mlp(a.H, [&](auto Hc, auto SAc, auto SVc) {
    mlp_softmax_aggregate_bwd_kernel<decltype(Hc)::value, decltype(SAc)::value, decltype(SVc)::value>
        <<<dot_grid(n_nodes), 256, 0, st>>>(a, alpha, keep, rp, n_nodes, work);
  });
  return check_cuda(cudaGetLastError(), "mlp_softmax_aggregate_bwd_kernel launch");
}
