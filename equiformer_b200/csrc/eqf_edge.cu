// eqf_edge.cu - edge-feature producers of the hot path (SURVEY.md rows a11, a12, f-2): one kernel for the edge geometry
// (edge vector, length, real spherical harmonics up to l = 4) with its first-order backward to the edge vector, and the
// exp-normal radial basis of the MD17 models.
//
// Reference work replaced:
//   nets/graph_attention_transformer.py:866-870        edge_vec = pos[src] - pos[dst]; o3.spherical_harmonics(l, edge_vec,
//                                                      normalize=True, normalization='component'); edge_vec.norm(dim=1)
//   nets/graph_attention_transformer_oc20.py:283-296   the same with the periodic image offsets added
//   nets/expnorm_rbf.py:11-33, 73-78                   CosineCutoff * exp(-beta (exp(-alpha d) - mean)^2)
//   nets/graph_attention_transformer.py:786-787,       RadialBasis(num_basis, cutoff, rbf={'name': 'spherical_bessel'})
//   ..._md17.py:179-180, equiformer_md17_dens.py:123   of ocpmodels 0.0.3 (gemnet/layers/radial_basis.py): polynomial
//                                                      envelope (p = 5) * sqrt(2 / c^3) sin(f_k d / c) / (d / c)
// One thread per edge for the geometry (a few hundred flops, ~100 bytes), one warp per edge row for the bases.  The
// harmonics follow e3nn's coupling recurrence  Y_{l+1,k} = sum_ji A_l[k,j,i] x_j Y_{l,i}  ('norm' normalisation, y polar,
// Y_1 = (x, y, z)); the host passes the coupling tensors A_1, A_2, A_3 (equiformer_b200/o3/sh.py computes them from the
// real Wigner 3j), so kernel and torch statement share one table.  Second derivatives (MD17 force training) go through the
// torch statement (ops._higher_order_grads), like the other fused pointwise ops.
#include <cuda_runtime.h>

#include <cstdint>

#include "eqf_common.cuh"

namespace eqf {

struct EdgeGeomArgs {
  const float* pos;            // [N, 3]
  const long long* src;        // [E]
  const long long* dst;        // [E]
  const float* offsets;        // optional [E, 3] added to pos[src] - pos[dst] (periodic images)
  const float* a1;             // coupling 1 -> 2: [5][3][3]
  const float* a2;             // coupling 2 -> 3: [7][3][5]
  const float* a3;             // coupling 3 -> 4: [9][3][7]
  long long E;
  int lmax;                    // 0 .. 4
  int n_sh;                    // (lmax + 1)^2
};

// forward: vec [E, 3], len [E], sh [E, n_sh] ('component' normalisation: Y_l * sqrt(2l+1)), harmonics of the UNIT vector
__global__ void __launch_bounds__(256) edge_geom_fwd_kernel(EdgeGeomArgs a, float* __restrict__ vec, float* __restrict__ len,
                                                            float* __restrict__ sh) {
  __shared__ float c1[45], c2[105], c3[189];
  for (int i = threadIdx.x; i < 45; i += blockDim.x) c1[i] = a.lmax >= 2 ? a.a1[i] : 0.f;
  for (int i = threadIdx.x; i < 105; i += blockDim.x) c2[i] = a.lmax >= 3 ? a.a2[i] : 0.f;
  for (int i = threadIdx.x; i < 189; i += blockDim.x) c3[i] = a.lmax >= 4 ? a.a3[i] : 0.f;
  __syncthreads();
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.E) return;
  const long long s = a.src[e], t = a.dst[e];
  float v[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) v[q] = __ldg(a.pos + 3 * s + q) - __ldg(a.pos + 3 * t + q) + (a.offsets ? __ldg(a.offsets + 3 * e + q) : 0.f);
  const float r = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  const float inv = 1.f / fmaxf(r, 1e-12f);          // F.normalize(eps = 1e-12)
  const float x[3] = {v[0] * inv, v[1] * inv, v[2] * inv};
#pragma unroll
  for (int q = 0; q < 3; ++q) vec[3 * e + q] = v[q];
  len[e] = r;
  float* o = sh + e * a.n_sh;
  o[0] = 1.f;
  if (a.lmax < 1) return;
  const float s3 = 1.7320508075688772f;
#pragma unroll
  for (int q = 0; q < 3; ++q) o[1 + q] = s3 * x[q];
  if (a.lmax < 2) return;
  float y2[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int i = 0; i < 3; ++i) acc = fmaf(c1[(k * 3 + j) * 3 + i] * x[j], x[i], acc);
    y2[k] = acc;
    o[4 + k] = 2.23606797749979f * acc;
  }
  if (a.lmax < 3) return;
  float y3[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int i = 0; i < 5; ++i) acc = fmaf(c2[(k * 3 + j) * 5 + i] * x[j], y2[i], acc);
    y3[k] = acc;
    o[9 + k] = 2.6457513110645907f * acc;
  }
  if (a.lmax < 4) return;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int i = 0; i < 7; ++i) acc = fmaf(c3[(k * 3 + j) * 7 + i] * x[j], y3[i], acc);
    o[16 + k] = 3.f * acc;
  }
}

// backward: g_vec [E, 3] from g_sh [E, n_sh] (may be NULL) and g_len [E] (may be NULL); reverse sweep through the recurrence
__global__ void __launch_bounds__(256) edge_geom_bwd_kernel(EdgeGeomArgs a, const float* __restrict__ vec,
                                                            const float* __restrict__ g_sh, const float* __restrict__ g_len,
                                                            float* __restrict__ g_vec) {
  __shared__ float c1[45], c2[105], c3[189];
  for (int i = threadIdx.x; i < 45; i += blockDim.x) c1[i] = a.lmax >= 2 ? a.a1[i] : 0.f;
  for (int i = threadIdx.x; i < 105; i += blockDim.x) c2[i] = a.lmax >= 3 ? a.a2[i] : 0.f;
  for (int i = threadIdx.x; i < 189; i += blockDim.x) c3[i] = a.lmax >= 4 ? a.a3[i] : 0.f;
  __syncthreads();
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.E) return;
  const float v[3] = {__ldg(vec + 3 * e), __ldg(vec + 3 * e + 1), __ldg(vec + 3 * e + 2)};
  const float r = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  const float inv = 1.f / fmaxf(r, 1e-12f);
  const float x[3] = {v[0] * inv, v[1] * inv, v[2] * inv};
  float xb[3] = {0.f, 0.f, 0.f};                       // adjoint of the unit vector
  if (g_sh != nullptr && a.lmax >= 1) {
    const float* g = g_sh + e * a.n_sh;
    float y2[5] = {0.f, 0.f, 0.f, 0.f, 0.f}, g1[3], g2[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    float y3[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, g3[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int q = 0; q < 3; ++q) g1[q] = 1.7320508075688772f * __ldg(g + 1 + q);
    if (a.lmax >= 2) {
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
          for (int i = 0; i < 3; ++i) acc = fmaf(c1[(k * 3 + j) * 3 + i] * x[j], x[i], acc);
        y2[k] = acc;
        g2[k] = 2.23606797749979f * __ldg(g + 4 + k);
      }
    }
    if (a.lmax >= 3) {
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
          for (int i = 0; i < 5; ++i) acc = fmaf(c2[(k * 3 + j) * 5 + i] * x[j], y2[i], acc);
        y3[k] = acc;
        g3[k] = 2.6457513110645907f * __ldg(g + 9 + k);
      }
    }
    if (a.lmax >= 4) {                                  // Y_4 = A_3 . (x (x) Y_3): adjoints of x and of Y_3
#pragma unroll 1                                        // one Y_4 component at a time (fully unrolled: 72 registers)
      for (int k = 0; k < 9; ++k) {
        const float gk = 3.f * __ldg(g + 16 + k);
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
          for (int i = 0; i < 7; ++i) {
            const float c = c3[(k * 3 + j) * 7 + i] * gk;
            xb[j] = fmaf(c, y3[i], xb[j]);
            g3[i] = fmaf(c, x[j], g3[i]);
          }
      }
    }
    if (a.lmax >= 3) {                                  // Y_3 = A_2 . (x (x) Y_2): adjoints of x and of Y_2
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        const float gk = g3[k];
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
          for (int i = 0; i < 5; ++i) {
            const float c = c2[(k * 3 + j) * 5 + i] * gk;
            xb[j] = fmaf(c, y2[i], xb[j]);
            g2[i] = fmaf(c, x[j], g2[i]);
          }
      }
    }
    if (a.lmax >= 2) {                                  // Y_2 = A_1 . (x (x) Y_1), Y_1 = x
#pragma unroll
      for (int k = 0; k < 5; ++k)
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            const float c = c1[(k * 3 + j) * 3 + i] * g2[k];
            xb[j] = fmaf(c, x[i], xb[j]);
            g1[i] = fmaf(c, x[j], g1[i]);
          }
    }
#pragma unroll
    for (int q = 0; q < 3; ++q) xb[q] += g1[q];
  }
  // x = v / max(r, eps): dv = (xb - (xb . x) x) / r  (for r > eps), plus the length's own gradient g_len * x
  const float dotp = xb[0] * x[0] + xb[1] * x[1] + xb[2] * x[2];
  const float gl = g_len != nullptr ? __ldg(g_len + e) : 0.f;
  const bool tiny = r <= 1e-12f;
#pragma unroll
  for (int q = 0; q < 3; ++q) g_vec[3 * e + q] = tiny ? xb[q] * inv : fmaf(xb[q] - dotp * x[q], inv, gl * x[q]);
}

// exp-normal radial basis: out[e, b] = cutoff(d_e) * exp(-beta_b (exp(-alpha d_e) - mean_b)^2), cutoff = 0.5 (cos(pi d / hi) + 1) [d < hi]
__global__ void __launch_bounds__(256) expnorm_fwd_kernel(const float* __restrict__ dist, const float* __restrict__ means,
                                                          const float* __restrict__ betas, float alpha, float hi, long long E,
                                                          int B, float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= E * B) return;
  const long long e = idx / B;
  const int b = (int)(idx - e * B);
  const float d = __ldg(dist + e);
  const float cut = d < hi ? 0.5f * (cosf(d * 3.14159265358979323846f / hi) + 1.f) : 0.f;
  const float u = expf(-alpha * d) - __ldg(means + b);
  out[idx] = cut * expf(-__ldg(betas + b) * u * u);
}

// g_dist[e] = sum_b g[e, b] d out[e, b] / d d_e   (one warp per edge)
__global__ void __launch_bounds__(256) expnorm_bwd_kernel(const float* __restrict__ dist, const float* __restrict__ means,
                                                          const float* __restrict__ betas, float alpha, float hi, long long E,
                                                          int B, const float* __restrict__ g, float* __restrict__ g_dist) {
  const long long e = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (e >= E) return;
  const int lane = threadIdx.x & 31;
  const float d = __ldg(dist + e);
  const float pi_hi = 3.14159265358979323846f / hi;
  const bool in = d < hi;
  const float cut = in ? 0.5f * (cosf(d * pi_hi) + 1.f) : 0.f;
  const float dcut = in ? -0.5f * pi_hi * sinf(d * pi_hi) : 0.f;
  const float ex = expf(-alpha * d);
  float acc = 0.f;
  for (int b = lane; b < B; b += 32) {
    const float u = ex - __ldg(means + b), beta = __ldg(betas + b);
    const float gauss = expf(-beta * u * u);
    // d/dd [cut * gauss] = dcut * gauss + cut * gauss * (-2 beta u) * (-alpha ex)
    acc = fmaf(__ldg(g + e * B + b), gauss * (dcut + cut * 2.f * beta * u * alpha * ex), acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) g_dist[e] = acc;
}

// spherical Bessel radial basis (B <= 128 functions, lane owns k = lane + 32 j): with x = d / c,
//   env(x) = 1 - 21 x^5 + 35 x^6 - 15 x^7 for x < 1, else 0;   out[e, k] = env(x) sqrt(2 / c^3) sin(f_k x) / x.
// d = 0 gives 0 / 0 = NaN, as in the reference; neighbour lists never contain a zero-length edge.  The argument f_k x reaches
// 128 pi for the MD17 configurations: the accurate sincosf, never the __sinf intrinsic.
constexpr int kBesselMaxB = 128;
constexpr int kBesselPerLane = kBesselMaxB / 32;

__device__ __forceinline__ void bessel_envelope(float x, float& env, float& denv) {
  const bool in = x < 1.f;
  const float x2 = x * x, x4 = x2 * x2;
  env = in ? 1.f + x4 * x * fmaf(x, fmaf(x, -15.f, 35.f), -21.f) : 0.f;
  denv = in ? x4 * fmaf(x, fmaf(x, -105.f, 210.f), -105.f) : 0.f;      // 5a x^4 + 6b x^5 + 7c x^6
}

__global__ void __launch_bounds__(256) bessel_fwd_kernel(const float* __restrict__ dist, const float* __restrict__ freq,
                                                         float inv_cut, float norm, long long E, int B,
                                                         float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = (long long)gridDim.x * 8;
  float f[kBesselPerLane];
#pragma unroll
  for (int j = 0; j < kBesselPerLane; ++j) f[j] = lane + 32 * j < B ? __ldg(freq + lane + 32 * j) : 0.f;
  for (long long e = warp; e < E; e += n_warps) {
    const float x = __ldg(dist + e) * inv_cut;
    float env, denv;
    bessel_envelope(x, env, denv);
    const float scale = env * norm / x;
#pragma unroll
    for (int j = 0; j < kBesselPerLane; ++j) {
      const int k = lane + 32 * j;
      if (k < B) out[e * B + k] = scale * sinf(f[j] * x);
    }
  }
}

// g_dist[e] = sum_k g[e, k] d out[e, k] / d d_e (skipped when g_dist is NULL) and per-CTA partial rows
// part[grid][B] of d <g, out> / d f_k = sum_e g[e, k] env norm cos(f_k x_e)
__global__ void __launch_bounds__(256) bessel_bwd_kernel(const float* __restrict__ dist, const float* __restrict__ freq,
                                                         float inv_cut, float norm, const float* __restrict__ g, long long E,
                                                         int B, float* __restrict__ g_dist, float* __restrict__ part) {
  __shared__ float sacc[kBesselMaxB];
  for (int i = threadIdx.x; i < B; i += blockDim.x) sacc[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = (long long)gridDim.x * 8;
  float f[kBesselPerLane], af[kBesselPerLane];
#pragma unroll
  for (int j = 0; j < kBesselPerLane; ++j) {
    f[j] = lane + 32 * j < B ? __ldg(freq + lane + 32 * j) : 0.f;
    af[j] = 0.f;
  }
  for (long long e = warp; e < E; e += n_warps) {
    const float x = __ldg(dist + e) * inv_cut;
    float env, denv;
    bessel_envelope(x, env, denv);
    const float inv_x = 1.f / x;
    float gx = 0.f;
#pragma unroll
    for (int j = 0; j < kBesselPerLane; ++j) {
      const int k = lane + 32 * j;
      if (k < B) {
        const float gk = __ldg(g + e * B + k);
        float s, c;
        sincosf(f[j] * x, &s, &c);
        af[j] = fmaf(gk, env * c, af[j]);
        // d/dx [env sin(f x) / x] = denv sin / x + env (f cos - sin / x) / x
        gx = fmaf(gk, fmaf(denv, s, env * fmaf(f[j], c, -s * inv_x)) * inv_x, gx);
      }
    }
    if (g_dist != nullptr) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) gx += __shfl_xor_sync(0xffffffffu, gx, o);
      if (lane == 0) g_dist[e] = gx * norm * inv_cut;
    }
  }
#pragma unroll
  for (int j = 0; j < kBesselPerLane; ++j)
    if (lane + 32 * j < B) atomicAdd(&sacc[lane + 32 * j], af[j] * norm);
  __syncthreads();
  for (int i = threadIdx.x; i < B; i += blockDim.x) part[(long long)blockIdx.x * B + i] = sacc[i];
}

}  // namespace eqf

using namespace eqf;

static int fill_geom(EdgeGeomArgs& a, const float* pos, const int64_t* src, const int64_t* dst, const float* offsets,
                     const float* a1, const float* a2, const float* a3, int64_t E, int32_t lmax, const char* who) {
  if (lmax < 0 || lmax > 4) { set_error(std::string(who) + ": lmax must be 0..4"); return EQF_ERR_UNSUPPORTED; }
  if (!pos || !src || !dst || (lmax >= 2 && !a1) || (lmax >= 3 && !a2) || (lmax >= 4 && !a3)) {
    set_error(std::string(who) + ": null pointer"); return EQF_ERR_INVALID;
  }
  a.pos = pos; a.src = reinterpret_cast<const long long*>(src); a.dst = reinterpret_cast<const long long*>(dst);
  a.offsets = offsets; a.a1 = a1; a.a2 = a2; a.a3 = a3; a.E = E; a.lmax = lmax; a.n_sh = (lmax + 1) * (lmax + 1);
  return EQF_OK;
}

extern "C" int eqf_edge_geom_fwd(const float* pos, const int64_t* src, const int64_t* dst, const float* offsets,
                                 const float* a1, const float* a2, const float* a3, int64_t E, int32_t lmax, float* vec,
                                 float* len, float* sh, void* stream) {
  if (E <= 0) return EQF_OK;
  EdgeGeomArgs a;
  int rc = fill_geom(a, pos, src, dst, offsets, a1, a2, a3, E, lmax, "eqf_edge_geom_fwd");
  if (rc != EQF_OK) return rc;
  if (!vec || !len || !sh) { set_error("eqf_edge_geom_fwd: null output"); return EQF_ERR_INVALID; }
  edge_geom_fwd_kernel<<<(unsigned)((E + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, vec, len, sh);
  return check_cuda(cudaGetLastError(), "edge_geom_fwd_kernel launch");
}

extern "C" int eqf_edge_geom_bwd(const float* vec, const float* a1, const float* a2, const float* a3, int64_t E,
                                 int32_t lmax, const float* g_sh, const float* g_len, float* g_vec, void* stream) {
  if (E <= 0) return EQF_OK;
  if (lmax < 0 || lmax > 4 || !vec || !g_vec || (lmax >= 2 && !a1) || (lmax >= 3 && !a2) || (lmax >= 4 && !a3)) {
    set_error("eqf_edge_geom_bwd: bad arguments"); return EQF_ERR_INVALID;
  }
  EdgeGeomArgs a;
  a.pos = nullptr; a.src = a.dst = nullptr; a.offsets = nullptr; a.a1 = a1; a.a2 = a2; a.a3 = a3; a.E = E; a.lmax = lmax;
  a.n_sh = (lmax + 1) * (lmax + 1);
  edge_geom_bwd_kernel<<<(unsigned)((E + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, vec, g_sh, g_len, g_vec);
  return check_cuda(cudaGetLastError(), "edge_geom_bwd_kernel launch");
}

extern "C" int eqf_expnorm_fwd(const float* dist, const float* means, const float* betas, float alpha, float cutoff_upper,
                               int64_t E, int32_t B, float* out, void* stream) {
  if (E <= 0 || B <= 0) return EQF_OK;
  if (!dist || !means || !betas || !out) { set_error("eqf_expnorm_fwd: null pointer"); return EQF_ERR_INVALID; }
  const long long n = E * B;
  expnorm_fwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(dist, means, betas, alpha, cutoff_upper, E, B, out);
  return check_cuda(cudaGetLastError(), "expnorm_fwd_kernel launch");
}

extern "C" int eqf_expnorm_bwd(const float* dist, const float* means, const float* betas, float alpha, float cutoff_upper,
                               int64_t E, int32_t B, const float* g, float* g_dist, void* stream) {
  if (E <= 0 || B <= 0) return EQF_OK;
  if (!dist || !means || !betas || !g || !g_dist) { set_error("eqf_expnorm_bwd: null pointer"); return EQF_ERR_INVALID; }
  expnorm_bwd_kernel<<<(unsigned)((E + 7) / 8), 256, 0, (cudaStream_t)stream>>>(dist, means, betas, alpha, cutoff_upper, E, B, g, g_dist);
  return check_cuda(cudaGetLastError(), "expnorm_bwd_kernel launch");
}

static int check_bessel(int32_t B, float cutoff, const char* who) {
  // B % 4 == 0 keeps the [E, B] output a legal TMA operand of the first-layer GEMM
  if (B < 1 || B > kBesselMaxB || B % 4 != 0) { set_error(std::string(who) + ": B must be a multiple of 4 in 4..128"); return EQF_ERR_UNSUPPORTED; }
  if (!(cutoff > 0.f)) { set_error(std::string(who) + ": cutoff must be positive"); return EQF_ERR_INVALID; }
  return EQF_OK;
}

extern "C" int eqf_bessel_fwd(const float* dist, const float* freq, float cutoff, int64_t E, int32_t B, float* out,
                              void* stream) {
  int rc = check_bessel(B, cutoff, "eqf_bessel_fwd");
  if (rc != EQF_OK || E <= 0) return rc;
  if (!dist || !freq || !out) { set_error("eqf_bessel_fwd: null pointer"); return EQF_ERR_INVALID; }
  bessel_fwd_kernel<<<eqf_pointwise_rows(E), 256, 0, (cudaStream_t)stream>>>(dist, freq, 1.f / cutoff,
                                                                            sqrtf(2.f / (cutoff * cutoff * cutoff)), E, B, out);
  return check_cuda(cudaGetLastError(), "bessel_fwd_kernel launch");
}

extern "C" int eqf_bessel_bwd(const float* dist, const float* freq, float cutoff, const float* g, int64_t E, int32_t B,
                              float* g_dist, float* part, void* stream) {
  int rc = check_bessel(B, cutoff, "eqf_bessel_bwd");
  if (rc != EQF_OK || E <= 0) return rc;
  if (!dist || !freq || !g || !part) { set_error("eqf_bessel_bwd: null pointer"); return EQF_ERR_INVALID; }
  bessel_bwd_kernel<<<eqf_pointwise_rows(E), 256, 0, (cudaStream_t)stream>>>(dist, freq, 1.f / cutoff,
                                                                            sqrtf(2.f / (cutoff * cutoff * cutoff)), g, E, B,
                                                                            g_dist, part);
  return check_cuda(cudaGetLastError(), "bessel_bwd_kernel launch");
}
