// eqf_graph.cu - neighbour list (radius graph) for the batched-molecule inputs of the hot path.
//
// Replaces the torch brute force of equiformer_b200/graph.py (itself a stand-in for torch_cluster.radius_graph as called
// at nets/graph_attention_transformer.py:866-867): same contract - edge (j -> i) iff batch[j] == batch[i], j != i (unless
// `loop`), |pos_j - pos_i|^2 < r^2, at most `max_neighbors` neighbours per centre, the first ones in index order; edges
// sorted by centre i (edge_dst ascending), neighbours j ascending inside a centre.  Two passes of one warp per centre
// over all candidate atoms (ordered 32-wide chunks, ballot + popc give the running rank): count -> (exclusive scan on
// the caller's side) -> fill.  O(N^2) pair tests like the stand-in, but without its [N, N] intermediates (distance
// matrix, mask, cumsum, nonzero): 2 324 atoms = 5.4 M tests, a few microseconds.
#include <cuda_runtime.h>

#include <cstdint>

#include "eqf_common.cuh"

namespace eqf {

template <bool FILL>
__global__ void __launch_bounds__(256) radius_graph_kernel(const float* __restrict__ pos, const long long* __restrict__ batch,
                                                           long long n, float r2, int loop, long long max_nb,
                                                           long long* __restrict__ deg, const long long* __restrict__ row_ptr,
                                                           long long* __restrict__ src, long long* __restrict__ dst) {
  const int lane = threadIdx.x & 31;
  const long long i = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= n) return;
  const float xi = __ldg(pos + 3 * i), yi = __ldg(pos + 3 * i + 1), zi = __ldg(pos + 3 * i + 2);
  const long long bi = batch ? __ldg(batch + i) : 0;
  long long count = 0;
  const long long base = FILL ? __ldg(row_ptr + i) : 0;
  for (long long j0 = 0; j0 < n && count < max_nb; j0 += 32) {
    const long long j = j0 + lane;
    bool hit = false;
    if (j < n) {
      const float dx = xi - __ldg(pos + 3 * j), dy = yi - __ldg(pos + 3 * j + 1), dz = zi - __ldg(pos + 3 * j + 2);
      // same arithmetic as the torch stand-in (separately rounded squares, left-to-right sum; no FMA contraction), so the
      // two agree on boundary pairs too
      const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      hit = d2 < r2 && (batch ? __ldg(batch + j) == bi : true) && (loop || j != i);
    }
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    const long long rank = count + __popc(m & ((1u << lane) - 1u));
    if (FILL && hit && rank < max_nb) {
      src[base + rank] = j;
      dst[base + rank] = i;
    }
    count += __popc(m);
  }
  if (!FILL && lane == 0) deg[i] = count < max_nb ? count : max_nb;
}

}  // namespace eqf

using namespace eqf;

// deg[i] = number of neighbours of centre i (capped at max_neighbors)
extern "C" int eqf_radius_graph_count(const float* pos, const int64_t* batch, int64_t n, float r_squared, int32_t loop,
                                      int64_t max_neighbors, int64_t* deg, void* stream) {
  if (n <= 0) return EQF_OK;
  if (!pos || !deg || max_neighbors < 0) { set_error("eqf_radius_graph_count: bad arguments"); return EQF_ERR_INVALID; }
  radius_graph_kernel<false><<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(
      pos, reinterpret_cast<const long long*>(batch), n, r_squared, loop, max_neighbors, reinterpret_cast<long long*>(deg), nullptr,
      nullptr, nullptr);
  return check_cuda(cudaGetLastError(), "radius_graph_kernel<count> launch");
}

// src / dst [row_ptr[n]] from the exclusive scan row_ptr[n + 1] of deg
extern "C" int eqf_radius_graph_fill(const float* pos, const int64_t* batch, int64_t n, float r_squared, int32_t loop,
                                     int64_t max_neighbors, const int64_t* row_ptr, int64_t* src, int64_t* dst, void* stream) {
  if (n <= 0) return EQF_OK;
  if (!pos || !row_ptr || !src || !dst) { set_error("eqf_radius_graph_fill: null pointer"); return EQF_ERR_INVALID; }
  radius_graph_kernel<true><<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(
      pos, reinterpret_cast<const long long*>(batch), n, r_squared, loop, max_neighbors, nullptr,
      reinterpret_cast<const long long*>(row_ptr), reinterpret_cast<long long*>(src), reinterpret_cast<long long*>(dst));
  return check_cuda(cudaGetLastError(), "radius_graph_kernel<fill> launch");
}

// ------------------------------------------------------------------------------------------------ periodic cells
// Neighbour list under periodic boundary conditions (what ocpmodels' radius_graph_pbc + get_pbc_distances give the OC20
// model at nets/graph_attention_transformer_oc20.py:267-302): edge (j, image c) -> i iff atoms i and j belong to the
// same frame and |pos_j + c . cell - pos_i| < r with (j, c) != (i, 0); images c in [-rep_a, rep_a] x [-rep_b, rep_b] x
// [-rep_c, rep_c] (the caller derives the repetitions from the cell heights and r, as ocpmodels does); the pair is kept
// when 1e-4 < distance^2 <= r^2 (ocpmodels' two masks).  One warp per
// centre walks the frame's atoms x images in a fixed order (atom ascending, image index ascending); ballot / popc ranks
// give each hit its slot: sorted by centre, deterministic.
namespace eqf {

template <bool FILL>
__global__ void __launch_bounds__(256) radius_graph_pbc_kernel(const float* __restrict__ pos, const long long* __restrict__ batch,
                                                               const long long* __restrict__ frame_ptr, const float* __restrict__ cell,
                                                               long long n, float r2, int rep_a, int rep_b, int rep_c,
                                                               long long* __restrict__ deg, const long long* __restrict__ row_ptr,
                                                               long long* __restrict__ src, long long* __restrict__ dst,
                                                               int* __restrict__ offs, float* __restrict__ dist2) {
  const int lane = threadIdx.x & 31;
  const long long i = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= n) return;
  const long long f = __ldg(batch + i);
  const long long j_begin = __ldg(frame_ptr + f), j_end = __ldg(frame_ptr + f + 1);
  const float* c = cell + 9 * f;             // rows = lattice vectors a, b, c
  float cm[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) cm[q] = __ldg(c + q);
  const float xi = __ldg(pos + 3 * i), yi = __ldg(pos + 3 * i + 1), zi = __ldg(pos + 3 * i + 2);
  const int na = 2 * rep_a + 1, nb = 2 * rep_b + 1, nc = 2 * rep_c + 1;
  const long long n_img = (long long)na * nb * nc;
  const long long total = (j_end - j_begin) * n_img;
  long long count = 0;
  const long long base = FILL ? __ldg(row_ptr + i) : 0;
  for (long long t0 = 0; t0 < total; t0 += 32) {
    const long long t = t0 + lane;
    bool hit = false;
    long long j = 0;
    int ia = 0, ib = 0, ic = 0;
    float d2 = 0.f;
    if (t < total) {
      j = j_begin + t / n_img;
      const int img = (int)(t % n_img);
      ia = img / (nb * nc) - rep_a;
      ib = (img / nc) % nb - rep_b;
      ic = img % nc - rep_c;
      // image offset ia a + ib b + ic c as separately rounded products summed in that order, the arithmetic of the torch
      // statement: left to the compiler the sum becomes an FMA chain, which rounds differently and so keeps or drops
      // some pairs within an ulp of r^2 that the statement decides the other way
      const float fa = (float)ia, fb = (float)ib, fc = (float)ic;
      const float ox = __fadd_rn(__fadd_rn(__fmul_rn(fa, cm[0]), __fmul_rn(fb, cm[3])), __fmul_rn(fc, cm[6]));
      const float oy = __fadd_rn(__fadd_rn(__fmul_rn(fa, cm[1]), __fmul_rn(fb, cm[4])), __fmul_rn(fc, cm[7]));
      const float oz = __fadd_rn(__fadd_rn(__fmul_rn(fa, cm[2]), __fmul_rn(fb, cm[5])), __fmul_rn(fc, cm[8]));
      const float dx = __ldg(pos + 3 * j) + ox - xi, dy = __ldg(pos + 3 * j + 1) + oy - yi, dz = __ldg(pos + 3 * j + 2) + oz - zi;
      d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      hit = d2 <= r2 && d2 > 1e-4f;          // ocpmodels' masks: distance_sqr <= r^2 and distance_sqr > 0.0001 (the atom itself)
    }
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (FILL && hit) {
      const long long slot = base + count + __popc(m & ((1u << lane) - 1u));
      src[slot] = j;
      dst[slot] = i;
      offs[3 * slot] = ia; offs[3 * slot + 1] = ib; offs[3 * slot + 2] = ic;
      dist2[slot] = d2;
    }
    count += __popc(m);
  }
  if (!FILL && lane == 0) deg[i] = count;
}

}  // namespace eqf

extern "C" int eqf_radius_graph_pbc_count(const float* pos, const int64_t* batch, const int64_t* frame_ptr, const float* cell,
                                          int64_t n, float r_squared, int32_t rep_a, int32_t rep_b, int32_t rep_c, int64_t* deg,
                                          void* stream) {
  if (n <= 0) return EQF_OK;
  if (!pos || !batch || !frame_ptr || !cell || !deg || rep_a < 0 || rep_b < 0 || rep_c < 0) {
    set_error("eqf_radius_graph_pbc_count: bad arguments"); return EQF_ERR_INVALID;
  }
  radius_graph_pbc_kernel<false><<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(
      pos, reinterpret_cast<const long long*>(batch), reinterpret_cast<const long long*>(frame_ptr), cell, n, r_squared, rep_a,
      rep_b, rep_c, reinterpret_cast<long long*>(deg), nullptr, nullptr, nullptr, nullptr, nullptr);
  return check_cuda(cudaGetLastError(), "radius_graph_pbc_kernel<count> launch");
}

extern "C" int eqf_radius_graph_pbc_fill(const float* pos, const int64_t* batch, const int64_t* frame_ptr, const float* cell,
                                         int64_t n, float r_squared, int32_t rep_a, int32_t rep_b, int32_t rep_c,
                                         const int64_t* row_ptr, int64_t* src, int64_t* dst, int32_t* cell_offsets, float* dist2,
                                         void* stream) {
  if (n <= 0) return EQF_OK;
  if (!pos || !batch || !frame_ptr || !cell || !row_ptr || !src || !dst || !cell_offsets || !dist2) {
    set_error("eqf_radius_graph_pbc_fill: null pointer"); return EQF_ERR_INVALID;
  }
  radius_graph_pbc_kernel<true><<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(
      pos, reinterpret_cast<const long long*>(batch), reinterpret_cast<const long long*>(frame_ptr), cell, n, r_squared, rep_a,
      rep_b, rep_c, nullptr, reinterpret_cast<const long long*>(row_ptr), reinterpret_cast<long long*>(src),
      reinterpret_cast<long long*>(dst), cell_offsets, dist2);
  return check_cuda(cudaGetLastError(), "radius_graph_pbc_kernel<fill> launch");
}
