// eqf_pointwise.cu - fused per-edge pointwise kernels around the GEMMs of the attention path (sm_90a).
//
// Reference work replaced:
//   * RadialProfile's hidden layers (nets/radial_func.py:24-35): LayerNorm -> SiLU on [E, 64] after each Linear -
//     eager: native_layer_norm + silu (+ in backward layer_norm_backward with its separate gamma/beta reduction)
//     -> ln_silu_{fwd,bwd}_kernel, one warp per row;
//   * the middle of GraphAttention.forward (nets/graph_attention_transformer.py:492-495,506-507): bias adds, the Gate
//     (SiLU on scalars, sigmoid gates x gated irreps, e3nn normalize2mom constants) and the attention logits
//     (SmoothLeakyReLU . alpha_dot) -> gate_logits_{fwd,bwd}_kernel, one warp per edge;
// all HBM-streaming: every input element is read once, every output written once.
#include "eqf_common.cuh"

namespace eqf {

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ------------------------------------------------------------------------------------------------ LayerNorm + SiLU
// y = silu(z), z = (x - mean) * rstd * gamma + beta ; C <= 32 * kMaxPerLane, one warp per row.  The kernels are
// instantiated for 2 / 4 / 8 columns per lane: at C = 64 (the radial MLP) the 8-column version carried 102 registers
// for six live arrays it did not need - 2 CTAs per SM and a latency-bound kernel.
constexpr int kMaxPerLane = 8;

template <int PER>
__global__ void __launch_bounds__(256) ln_silu_fwd_kernel(const float* __restrict__ x, const float* __restrict__ bias,
                                                          const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, float eps, long long R, int C,
                                                          float* __restrict__ y, float* __restrict__ mean,
                                                          float* __restrict__ rstd) {
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = (long long)gridDim.x * 8;
  for (long long r = warp; r < R; r += n_warps) {
    float v[PER];
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int c = lane + 32 * q;
      v[q] = (c < C) ? __ldg(x + r * C + c) + (bias ? __ldg(bias + c) : 0.f) : 0.f;   // bias of the preceding Linear
      s += v[q];
    }
    const float m = wsum(s) / C;
    float ss = 0.f;
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int c = lane + 32 * q;
      const float d = (c < C) ? v[q] - m : 0.f;
      ss += d * d;
    }
    const float rs = rsqrtf(wsum(ss) / C + eps);
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int c = lane + 32 * q;
      if (c < C) {
        const float z = (v[q] - m) * rs * __ldg(gamma + c) + __ldg(beta + c);
        y[r * C + c] = z * sigmoidf_(z);
      }
    }
    if (lane == 0) { mean[r] = m; rstd[r] = rs; }
  }
}

// gx, and per-CTA partial sums [gridDim.x][3C] = d gamma | d beta | d bias (= column sums of gx)
template <int PER>
__global__ void __launch_bounds__(256) ln_silu_bwd_kernel(const float* __restrict__ x, const float* __restrict__ bias,
                                                          const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, const float* __restrict__ mean,
                                                          const float* __restrict__ rstd, const float* __restrict__ gy,
                                                          long long R, int C, float* __restrict__ gx,
                                                          float* __restrict__ part) {
  __shared__ float sg[32 * PER], sb[32 * PER], sx[32 * PER];
  for (int i = threadIdx.x; i < 32 * PER; i += blockDim.x) { sg[i] = 0.f; sb[i] = 0.f; sx[i] = 0.f; }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = (long long)gridDim.x * 8;
  float ag[PER], ab[PER], ax[PER];
#pragma unroll
  for (int q = 0; q < PER; ++q) { ag[q] = 0.f; ab[q] = 0.f; ax[q] = 0.f; }
  for (long long r = warp; r < R; r += n_warps) {
    const float m = __ldg(mean + r), rs = __ldg(rstd + r);
    float xh[PER], gz[PER];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int c = lane + 32 * q;
      xh[q] = 0.f; gz[q] = 0.f;
      if (c < C) {
        const float g = __ldg(gamma + c);
        xh[q] = (__ldg(x + r * C + c) + (bias ? __ldg(bias + c) : 0.f) - m) * rs;
        const float z = xh[q] * g + __ldg(beta + c);
        const float sg_ = sigmoidf_(z);
        const float dz = __ldg(gy + r * C + c) * (sg_ * (1.f + z * (1.f - sg_)));   // d silu / dz
        ag[q] += dz * xh[q];
        ab[q] += dz;
        gz[q] = dz * g;
        s1 += gz[q];
        s2 += gz[q] * xh[q];
      }
    }
    s1 = wsum(s1) / C;
    s2 = wsum(s2) / C;
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int c = lane + 32 * q;
      if (c < C) {
        const float v = rs * (gz[q] - s1 - xh[q] * s2);
        gx[r * C + c] = v;
        ax[q] += v;
      }
    }
  }
#pragma unroll
  for (int q = 0; q < PER; ++q) {
    const int c = lane + 32 * q;
    if (c < C) { atomicAdd(&sg[c], ag[q]); atomicAdd(&sb[c], ab[q]); atomicAdd(&sx[c], ax[q]); }
  }
  __syncthreads();
  float* row = part + (long long)blockIdx.x * 3 * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    row[c] = sg[c];
    row[C + c] = sb[c];
    row[2 * C + c] = sx[c];
  }
}

// C == 64 (the radial MLP): half a warp per row, one float4 per lane - two rows in flight per warp, a quarter of the
// memory instructions and 4-step reductions; the generic kernels above are latency bound at this width.
__device__ __forceinline__ float hsum16(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(256) ln_silu_fwd64_kernel(const float* __restrict__ x, const float* __restrict__ bias,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            float eps, long long R, float* __restrict__ y,
                                                            float* __restrict__ mean, float* __restrict__ rstd) {
  const int lane = threadIdx.x & 31, sub = lane & 15;
  const long long pair = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_pairs = (long long)gridDim.x * 8;
  const float4 g4 = __ldg(reinterpret_cast<const float4*>(gamma) + sub), b4 = __ldg(reinterpret_cast<const float4*>(beta) + sub);
  const float4 p4 = bias ? __ldg(reinterpret_cast<const float4*>(bias) + sub) : make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long r = pair * 2 + (lane >> 4); r < R + (lane >> 4); r += n_pairs * 2) {   // both halves iterate together
    const bool ok = r < R;
    float4 v = ok ? __ldg(reinterpret_cast<const float4*>(x + r * 64) + sub) : make_float4(0.f, 0.f, 0.f, 0.f);
    v.x += p4.x; v.y += p4.y; v.z += p4.z; v.w += p4.w;
    const float m = hsum16(v.x + v.y + v.z + v.w) * (1.f / 64.f);
    const float dx = v.x - m, dy = v.y - m, dz = v.z - m, dw = v.w - m;
    const float rs = rsqrtf(hsum16(dx * dx + dy * dy + dz * dz + dw * dw) * (1.f / 64.f) + eps);
    if (ok) {
      const float zx = dx * rs * g4.x + b4.x, zy = dy * rs * g4.y + b4.y, zz = dz * rs * g4.z + b4.z, zw = dw * rs * g4.w + b4.w;
      reinterpret_cast<float4*>(y + r * 64)[sub] = make_float4(zx * sigmoidf_(zx), zy * sigmoidf_(zy), zz * sigmoidf_(zz), zw * sigmoidf_(zw));
      if (sub == 0) { mean[r] = m; rstd[r] = rs; }
    }
  }
}

__global__ void __launch_bounds__(256) ln_silu_bwd64_kernel(const float* __restrict__ x, const float* __restrict__ bias,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            const float* __restrict__ mean, const float* __restrict__ rstd,
                                                            const float* __restrict__ gy, long long R, float* __restrict__ gx,
                                                            float* __restrict__ part) {
  __shared__ float sacc[3 * 64];
  for (int i = threadIdx.x; i < 3 * 64; i += blockDim.x) sacc[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31, sub = lane & 15;
  const long long pair = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_pairs = (long long)gridDim.x * 8;
  const float4 g4 = __ldg(reinterpret_cast<const float4*>(gamma) + sub), b4 = __ldg(reinterpret_cast<const float4*>(beta) + sub);
  const float4 p4 = bias ? __ldg(reinterpret_cast<const float4*>(bias) + sub) : make_float4(0.f, 0.f, 0.f, 0.f);
  float ag[4] = {0.f, 0.f, 0.f, 0.f}, ab[4] = {0.f, 0.f, 0.f, 0.f}, ax[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long r = pair * 2 + (lane >> 4); r < R + (lane >> 4); r += n_pairs * 2) {
    const bool ok = r < R;
    const float m = ok ? __ldg(mean + r) : 0.f, rs = ok ? __ldg(rstd + r) : 0.f;
    const float4 xv = ok ? __ldg(reinterpret_cast<const float4*>(x + r * 64) + sub) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 gv = ok ? __ldg(reinterpret_cast<const float4*>(gy + r * 64) + sub) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float xs[4] = {xv.x + p4.x, xv.y + p4.y, xv.z + p4.z, xv.w + p4.w};
    const float gs[4] = {gv.x, gv.y, gv.z, gv.w};
    const float gm[4] = {g4.x, g4.y, g4.z, g4.w}, bt[4] = {b4.x, b4.y, b4.z, b4.w};
    float xh[4], gz[4], s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      xh[q] = (xs[q] - m) * rs;
      const float z = xh[q] * gm[q] + bt[q];
      const float sg_ = sigmoidf_(z);
      const float dz = gs[q] * (sg_ * (1.f + z * (1.f - sg_)));
      ag[q] += dz * xh[q];
      ab[q] += dz;
      gz[q] = dz * gm[q];
      s1 += gz[q];
      s2 += gz[q] * xh[q];
    }
    s1 = hsum16(s1) * (1.f / 64.f);
    s2 = hsum16(s2) * (1.f / 64.f);
    float o[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) { o[q] = rs * (gz[q] - s1 - xh[q] * s2); ax[q] += o[q]; }
    if (ok) reinterpret_cast<float4*>(gx + r * 64)[sub] = make_float4(o[0], o[1], o[2], o[3]);
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    atomicAdd(&sacc[4 * sub + q], ag[q]);
    atomicAdd(&sacc[64 + 4 * sub + q], ab[q]);
    atomicAdd(&sacc[128 + 4 * sub + q], ax[q]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * 64; i += blockDim.x) part[(long long)blockIdx.x * 192 + i] = sacc[i];
}

// ------------------------------------------------------------------------------------------------ Gaussian radial basis
// rbf[e, k] = exp(-z^2 / 2) / (a s_k),  z = (w d_e / cutoff + b - mean_k) / s_k,  s_k = |std_k| + 1e-5,  a = sqrt(2 * 3.14159)
// (GaussianRadialBasisLayer, nets/gaussian_rbf.py:5-40; the truncated pi is the reference's).  One warp per edge, K = 128
// basis functions as one float4 per lane; the eager version is ~5 elementwise launches forward and ~15 backward (four of
// them [E, 128] column reductions) on the same [E, 128] tensor.
constexpr float kRbfA = 2.5066272160f;   // sqrt(2 * 3.14159): the reference truncates pi

__global__ void __launch_bounds__(256) rbf_fwd_kernel(const float* __restrict__ dist, const float* __restrict__ mean,
                                                      const float* __restrict__ std, const float* __restrict__ wp,
                                                      const float* __restrict__ bp, float inv_cut,
                                                      long long E, float* __restrict__ out) {
  const float w = __ldg(wp), b = __ldg(bp);       // [1, 1] parameters: read on the device (no host synchronisation)
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = (long long)gridDim.x * 8;
  const float4 m4 = __ldg(reinterpret_cast<const float4*>(mean) + lane);
  float4 s4 = __ldg(reinterpret_cast<const float4*>(std) + lane);
  s4 = make_float4(fabsf(s4.x) + 1e-5f, fabsf(s4.y) + 1e-5f, fabsf(s4.z) + 1e-5f, fabsf(s4.w) + 1e-5f);
  for (long long e = warp; e < E; e += n_warps) {
    const float x = w * (__ldg(dist + e) * inv_cut) + b;
    const float zx = (x - m4.x) / s4.x, zy = (x - m4.y) / s4.y, zz = (x - m4.z) / s4.z, zw = (x - m4.w) / s4.w;
    reinterpret_cast<float4*>(out + e * 128)[lane] =
        make_float4(expf(-0.5f * zx * zx) / (kRbfA * s4.x), expf(-0.5f * zy * zy) / (kRbfA * s4.y),
                    expf(-0.5f * zz * zz) / (kRbfA * s4.z), expf(-0.5f * zw * zw) / (kRbfA * s4.w));
  }
}

// g_dist[e] and per-CTA partial rows part[grid][258] = d mean (128) | d std (128) | d w | d b
__global__ void __launch_bounds__(256) rbf_bwd_kernel(const float* __restrict__ dist, const float* __restrict__ mean,
                                                      const float* __restrict__ std, const float* __restrict__ wp,
                                                      const float* __restrict__ bp, float inv_cut,
                                                      const float* __restrict__ g, long long E, float* __restrict__ g_dist,
                                                      float* __restrict__ part) {
  const float w = __ldg(wp), b = __ldg(bp);
  __shared__ float sacc[258];
  for (int i = threadIdx.x; i < 258; i += blockDim.x) sacc[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = (long long)gridDim.x * 8;
  const float4 m4 = __ldg(reinterpret_cast<const float4*>(mean) + lane);
  const float4 r4 = __ldg(reinterpret_cast<const float4*>(std) + lane);
  const float mm[4] = {m4.x, m4.y, m4.z, m4.w};
  const float raw[4] = {r4.x, r4.y, r4.z, r4.w};
  float ss[4], am[4] = {0.f, 0.f, 0.f, 0.f}, as[4] = {0.f, 0.f, 0.f, 0.f}, aw = 0.f, ab = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) ss[q] = fabsf(raw[q]) + 1e-5f;
  for (long long e = warp; e < E; e += n_warps) {
    const float d = __ldg(dist + e) * inv_cut;
    const float x = w * d + b;
    const float4 g4 = __ldg(reinterpret_cast<const float4*>(g + e * 128) + lane);
    const float gg[4] = {g4.x, g4.y, g4.z, g4.w};
    float gx = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float z = (x - mm[q]) / ss[q];
      const float o = expf(-0.5f * z * z) / (kRbfA * ss[q]);
      const float t = gg[q] * o / ss[q];          // g * out / s
      gx -= t * z;                                 // d out / d x = -z out / s
      am[q] += t * z;                              // d out / d mean = +z out / s
      as[q] += t * (z * z - 1.f);                  // d out / d s = out (z^2 - 1) / s
    }
    gx = wsum(gx);
    if (lane == 0) {
      g_dist[e] = gx * w * inv_cut;
      aw += gx * d;
      ab += gx;
    }
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    atomicAdd(&sacc[4 * lane + q], am[q]);
    atomicAdd(&sacc[128 + 4 * lane + q], as[q] * (raw[q] < 0.f ? -1.f : 1.f));     // d|std| / d std
  }
  if (lane == 0) { atomicAdd(&sacc[256], aw); atomicAdd(&sacc[257], ab); }
  __syncthreads();
  for (int i = threadIdx.x; i < 258; i += blockDim.x) part[(long long)blockIdx.x * 258 + i] = sacc[i];
}

// ------------------------------------------------------------------------------------------------ gate + logits
// Inputs (planar): t0 [E, A0 + S + Gt]  = [alpha pre-activations | scalars | gates]   (biases already added)
//                  gated blocks g_b [E, d_b, C_b] (b < n_gated), sum_b C_b == Gt, gates consumed in block order
// Outputs: z [E, H] attention logits; v0 [E, S]; v_b [E, d_b, C_b]
struct GateArgs {
  const float* t0;
  const float* gated[EQF_MAX_BLOCKS];
  float* v0;
  float* vout[EQF_MAX_BLOCKS];
  float* z;
  const float* alpha_dot;  // [H, A0/H]
  const float* bias;       // optional [A0 + S + Gt], added to t0 on the fly
  // backward
  const float* gz;               // [E, H]
  const float* gv0;              // [E, S]
  const float* gvout[EQF_MAX_BLOCKS];
  float* gt0;                    // [E, A0 + S + Gt]
  float* ggated[EQF_MAX_BLOCKS];
  float* gdot_part;              // [grid, A0]
  int n_gated, A0, S, Gt, H;
  int d[EQF_MAX_BLOCKS], C[EQF_MAX_BLOCKS];
  float c_silu, c_sig, c_slr, slope;
  long long E;
};

__global__ void __launch_bounds__(256) gate_logits_fwd_kernel(GateArgs a) {
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = (long long)gridDim.x * 8;
  const int T0 = a.A0 + a.S + a.Gt, ah = a.A0 / a.H;
  const float k1 = 0.5f * (1.f + a.slope), k2 = 0.5f * (1.f - a.slope);
  const float* bs = a.bias;
  for (long long e = warp; e < a.E; e += n_warps) {
    const float* t = a.t0 + e * T0;
    // logits: z[h] = sum_k c_slr * slr(t[h*ah + k]) * alpha_dot[h, k]
    for (int h = 0; h < a.H; ++h) {
      float acc = 0.f;
      for (int k = lane; k < ah; k += 32) {
        const float xv = __ldg(t + h * ah + k) + (bs ? __ldg(bs + h * ah + k) : 0.f);
        const float s = sigmoidf_(xv);
        acc = fmaf(a.c_slr * (k1 * xv + k2 * xv * (2.f * s - 1.f)), __ldg(a.alpha_dot + h * ah + k), acc);
      }
      acc = wsum(acc);
      if (lane == 0) a.z[e * a.H + h] = acc;
    }
    for (int c = lane; c < a.S; c += 32) {
      const float xv = __ldg(t + a.A0 + c) + (bs ? __ldg(bs + a.A0 + c) : 0.f);
      a.v0[e * a.S + c] = a.c_silu * xv * sigmoidf_(xv);
    }
    int goff = a.A0 + a.S;
    for (int b = 0; b < a.n_gated; ++b) {
      const int C = a.C[b], d = a.d[b];
      const float* gb = a.gated[b] + e * d * C;
      float* vb = a.vout[b] + e * d * C;
      for (int c = lane; c < C; c += 32) {
        const float gate = a.c_sig * sigmoidf_(__ldg(t + goff + c) + (bs ? __ldg(bs + goff + c) : 0.f));
        for (int i = 0; i < d; ++i) vb[i * C + c] = __ldg(gb + i * C + c) * gate;
      }
      goff += C;
    }
  }
}

__global__ void __launch_bounds__(256) gate_logits_bwd_kernel(GateArgs a) {
  extern __shared__ float sdot[];  // [A0]
  for (int i = threadIdx.x; i < a.A0; i += blockDim.x) sdot[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = (long long)gridDim.x * 8;
  const int T0 = a.A0 + a.S + a.Gt, ah = a.A0 / a.H;
  const float k1 = 0.5f * (1.f + a.slope), k2 = 0.5f * (1.f - a.slope);
  const float* bs = a.bias;
  const bool reg_acc = (ah <= 32 && a.H <= EQF_MAX_HEADS);   // alpha_dot gradient in registers (no shared atomics per edge)
  float adot[EQF_MAX_HEADS];
#pragma unroll
  for (int h = 0; h < EQF_MAX_HEADS; ++h) adot[h] = 0.f;
  for (long long e = warp; e < a.E; e += n_warps) {
    const float* t = a.t0 + e * T0;
    float* gt = a.gt0 + e * T0;
#pragma unroll
    for (int h = 0; h < EQF_MAX_HEADS; ++h) {
      if (h < a.H) {
        const float gzh = __ldg(a.gz + e * a.H + h);
        for (int k = lane; k < ah; k += 32) {
          const float xv = __ldg(t + h * ah + k) + (bs ? __ldg(bs + h * ah + k) : 0.f);
          const float s = sigmoidf_(xv);
          const float act = a.c_slr * (k1 * xv + k2 * xv * (2.f * s - 1.f));
          const float dact = a.c_slr * (k1 + k2 * ((2.f * s - 1.f) + 2.f * xv * s * (1.f - s)));
          const float ad = __ldg(a.alpha_dot + h * ah + k);
          gt[h * ah + k] = gzh * ad * dact;
          if (reg_acc) adot[h] += gzh * act;
          else atomicAdd(&sdot[h * ah + k], gzh * act);
        }
      }
    }
    for (int c = lane; c < a.S; c += 32) {
      const float xv = __ldg(t + a.A0 + c) + (bs ? __ldg(bs + a.A0 + c) : 0.f);
      const float s = sigmoidf_(xv);
      gt[a.A0 + c] = __ldg(a.gv0 + e * a.S + c) * a.c_silu * (s * (1.f + xv * (1.f - s)));
    }
    int goff = a.A0 + a.S;
    for (int b = 0; b < a.n_gated; ++b) {
      const int C = a.C[b], d = a.d[b];
      const float* gb = a.gated[b] + e * d * C;
      const float* gvb = a.gvout[b] + e * d * C;
      float* ggb = a.ggated[b] + e * d * C;
      for (int c = lane; c < C; c += 32) {
        const float s = sigmoidf_(__ldg(t + goff + c) + (bs ? __ldg(bs + goff + c) : 0.f));
        const float gate = a.c_sig * s;
        float acc = 0.f;
        for (int i = 0; i < d; ++i) {
          const float gv = __ldg(gvb + i * C + c);
          ggb[i * C + c] = gv * gate;
          acc = fmaf(gv, __ldg(gb + i * C + c), acc);
        }
        gt[goff + c] = acc * a.c_sig * s * (1.f - s);
      }
      goff += C;
    }
  }
  if (reg_acc && lane < ah) {
#pragma unroll
    for (int h = 0; h < EQF_MAX_HEADS; ++h)
      if (h < a.H) atomicAdd(&sdot[h * ah + lane], adot[h]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < a.A0; i += blockDim.x) a.gdot_part[(long long)blockIdx.x * a.A0 + i] = sdot[i];
}

// ------------------------------------------------------------------------------------------------ 128-bit gate/logits
// Same math, float4 lanes: requires A0, S, every C and A0/H to be multiples of 4 and (A0/H)/4 a power of two <= 32
// (all shipped configs).  Phase 1: lanes over alpha float4s (head partial sums combined with shuffles); phase 2: lanes
// over scalar float4s; phase 3: lanes over gate float4s, each lane walking the 2l+1 components of its gated channels.
__device__ __forceinline__ float4 ld4p(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void st4p(float* p, const float4& v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 add4(const float4& a, const float4& b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

struct GateBlockRef { int b; int c; };
__device__ __forceinline__ GateBlockRef gate_block(const GateArgs& a, int q4) {   // q4: float4 index inside the gates
  int b = 0, c = q4 * 4;
  while (b + 1 < a.n_gated && c >= a.C[b]) { c -= a.C[b]; ++b; }
  return {b, c};
}

__device__ __forceinline__ float slr_act(float x, float k1, float k2, float c) {
  const float s = sigmoidf_(x);
  return c * (k1 * x + k2 * x * (2.f * s - 1.f));
}
__device__ __forceinline__ float slr_dact(float x, float k1, float k2, float c) {
  const float s = sigmoidf_(x);
  return c * (k1 + k2 * ((2.f * s - 1.f) + 2.f * x * s * (1.f - s)));
}

__global__ void __launch_bounds__(256) gate_logits_fwd_vec_kernel(GateArgs a) {
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = (long long)gridDim.x * 8;
  const int T0 = a.A0 + a.S + a.Gt, ah = a.A0 / a.H, lph = ah / 4;   // lanes per head
  const float k1 = 0.5f * (1.f + a.slope), k2 = 0.5f * (1.f - a.slope);
  const float* bs = a.bias;
  for (long long e = warp; e < a.E; e += n_warps) {
    const float* t = a.t0 + e * T0;
    for (int q = lane; q < a.A0 / 4; q += 32) {           // ---- logits
      float4 x = ld4p(t + 4 * q);
      if (bs) x = add4(x, ld4p(bs + 4 * q));
      const float4 ad = ld4p(a.alpha_dot + 4 * q);
      float p = slr_act(x.x, k1, k2, a.c_slr) * ad.x + slr_act(x.y, k1, k2, a.c_slr) * ad.y +
                slr_act(x.z, k1, k2, a.c_slr) * ad.z + slr_act(x.w, k1, k2, a.c_slr) * ad.w;
      for (int o = lph >> 1; o > 0; o >>= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
      if ((q % lph) == 0) a.z[e * a.H + q / lph] = p;
    }
    for (int q = lane; q < a.S / 4; q += 32) {            // ---- scalars
      float4 x = ld4p(t + a.A0 + 4 * q);
      if (bs) x = add4(x, ld4p(bs + a.A0 + 4 * q));
      st4p(a.v0 + e * a.S + 4 * q, make_float4(a.c_silu * x.x * sigmoidf_(x.x), a.c_silu * x.y * sigmoidf_(x.y),
                                               a.c_silu * x.z * sigmoidf_(x.z), a.c_silu * x.w * sigmoidf_(x.w)));
    }
    for (int q = lane; q < a.Gt / 4; q += 32) {           // ---- gates x gated irreps
      float4 x = ld4p(t + a.A0 + a.S + 4 * q);
      if (bs) x = add4(x, ld4p(bs + a.A0 + a.S + 4 * q));
      const float4 gate = make_float4(a.c_sig * sigmoidf_(x.x), a.c_sig * sigmoidf_(x.y), a.c_sig * sigmoidf_(x.z),
                                      a.c_sig * sigmoidf_(x.w));
      const GateBlockRef r = gate_block(a, q);
      const int C = a.C[r.b], d = a.d[r.b];
      const float* gb = a.gated[r.b] + e * d * C + r.c;
      float* vb = a.vout[r.b] + e * d * C + r.c;
      for (int i = 0; i < d; ++i) {
        const float4 g = ld4p(gb + i * C);
        st4p(vb + i * C, make_float4(g.x * gate.x, g.y * gate.y, g.z * gate.z, g.w * gate.w));
      }
    }
  }
}

__global__ void __launch_bounds__(256) gate_logits_bwd_vec_kernel(GateArgs a) {
  extern __shared__ float sdot[];  // [A0]
  for (int i = threadIdx.x; i < a.A0; i += blockDim.x) sdot[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = (long long)gridDim.x * 8;
  const int T0 = a.A0 + a.S + a.Gt, ah = a.A0 / a.H, lph = ah / 4;
  const float k1 = 0.5f * (1.f + a.slope), k2 = 0.5f * (1.f - a.slope);
  const float* bs = a.bias;
  float4 adot = make_float4(0.f, 0.f, 0.f, 0.f);       // alpha_dot gradient of this lane's four (h, k) (A0/4 <= 32 lanes)
  const bool reg_acc = a.A0 / 4 <= 32;
  for (long long e = warp; e < a.E; e += n_warps) {
    const float* t = a.t0 + e * T0;
    float* gt = a.gt0 + e * T0;
    for (int q = lane; q < a.A0 / 4; q += 32) {
      float4 x = ld4p(t + 4 * q);
      if (bs) x = add4(x, ld4p(bs + 4 * q));
      const float4 ad = ld4p(a.alpha_dot + 4 * q);
      const float gzh = __ldg(a.gz + e * a.H + q / lph);
      st4p(gt + 4 * q, make_float4(gzh * ad.x * slr_dact(x.x, k1, k2, a.c_slr), gzh * ad.y * slr_dact(x.y, k1, k2, a.c_slr),
                                   gzh * ad.z * slr_dact(x.z, k1, k2, a.c_slr), gzh * ad.w * slr_dact(x.w, k1, k2, a.c_slr)));
      const float4 act = make_float4(gzh * slr_act(x.x, k1, k2, a.c_slr), gzh * slr_act(x.y, k1, k2, a.c_slr),
                                     gzh * slr_act(x.z, k1, k2, a.c_slr), gzh * slr_act(x.w, k1, k2, a.c_slr));
      if (reg_acc) adot = add4(adot, act);
      else { atomicAdd(&sdot[4 * q], act.x); atomicAdd(&sdot[4 * q + 1], act.y); atomicAdd(&sdot[4 * q + 2], act.z); atomicAdd(&sdot[4 * q + 3], act.w); }
    }
    for (int q = lane; q < a.S / 4; q += 32) {
      float4 x = ld4p(t + a.A0 + 4 * q);
      if (bs) x = add4(x, ld4p(bs + a.A0 + 4 * q));
      const float4 gv = ld4p(a.gv0 + e * a.S + 4 * q);
      const float sx = sigmoidf_(x.x), sy = sigmoidf_(x.y), sz = sigmoidf_(x.z), sw = sigmoidf_(x.w);
      st4p(gt + a.A0 + 4 * q, make_float4(gv.x * a.c_silu * sx * (1.f + x.x * (1.f - sx)), gv.y * a.c_silu * sy * (1.f + x.y * (1.f - sy)),
                                          gv.z * a.c_silu * sz * (1.f + x.z * (1.f - sz)), gv.w * a.c_silu * sw * (1.f + x.w * (1.f - sw))));
    }
    for (int q = lane; q < a.Gt / 4; q += 32) {
      float4 x = ld4p(t + a.A0 + a.S + 4 * q);
      if (bs) x = add4(x, ld4p(bs + a.A0 + a.S + 4 * q));
      const float sx = sigmoidf_(x.x), sy = sigmoidf_(x.y), sz = sigmoidf_(x.z), sw = sigmoidf_(x.w);
      const float4 gate = make_float4(a.c_sig * sx, a.c_sig * sy, a.c_sig * sz, a.c_sig * sw);
      const GateBlockRef r = gate_block(a, q);
      const int C = a.C[r.b], d = a.d[r.b];
      const float* gb = a.gated[r.b] + e * d * C + r.c;
      const float* gvb = a.gvout[r.b] + e * d * C + r.c;
      float* ggb = a.ggated[r.b] + e * d * C + r.c;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int i = 0; i < d; ++i) {
        const float4 gv = ld4p(gvb + i * C), g = ld4p(gb + i * C);
        st4p(ggb + i * C, make_float4(gv.x * gate.x, gv.y * gate.y, gv.z * gate.z, gv.w * gate.w));
        acc.x = fmaf(gv.x, g.x, acc.x); acc.y = fmaf(gv.y, g.y, acc.y); acc.z = fmaf(gv.z, g.z, acc.z); acc.w = fmaf(gv.w, g.w, acc.w);
      }
      st4p(gt + a.A0 + a.S + 4 * q, make_float4(acc.x * a.c_sig * sx * (1.f - sx), acc.y * a.c_sig * sy * (1.f - sy),
                                                acc.z * a.c_sig * sz * (1.f - sz), acc.w * a.c_sig * sw * (1.f - sw)));
    }
  }
  if (reg_acc && lane < a.A0 / 4) {
    atomicAdd(&sdot[4 * lane], adot.x); atomicAdd(&sdot[4 * lane + 1], adot.y);
    atomicAdd(&sdot[4 * lane + 2], adot.z); atomicAdd(&sdot[4 * lane + 3], adot.w);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < a.A0; i += blockDim.x) a.gdot_part[(long long)blockIdx.x * a.A0 + i] = sdot[i];
}

static bool gate_vec_ok(const GateArgs& a) {
  if (a.S % 4) return false;
  for (int b = 0; b < a.n_gated; ++b) if (a.C[b] % 4) return false;
  if (a.A0 == 0) return true;                           // gate-only use (FFN): the logits loops do not run at all
  if (a.A0 % 4 || (a.A0 / a.H) % 4) return false;
  const int lph = a.A0 / a.H / 4;
  if (lph < 1 || lph > 32 || (lph & (lph - 1))) return false;
  if (lph > 1 && (a.A0 / 4) % 32 != 0) return false;   // head sums use full-warp shuffles: every lane must take part
  return true;
}

// ------------------------------------------------------------------------------------------------ column sum
// out[c] = sum_r x[r, c]: bias / offset gradients (sum over all edges), reduction of per-CTA partial rows and of the
// sliced weight-gradient partials (torch's reduce_kernel runs the narrow ones on a single CTA).  Threads run along the columns (coalesced,
// float4 when aligned), rows are split over blockIdx.y; the last CTA to finish a column tile adds the partial rows in
// a fixed order (deterministic) and resets the tile's counter, so the buffer is reusable without a memset.
template <int VEC>
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ x, long long rows, long long cols, long long ld,
                                                     float* __restrict__ out, float* __restrict__ part,
                                                     unsigned int* __restrict__ counters) {
  __shared__ float red[8][32 * VEC];
  __shared__ bool last;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const long long c0 = ((long long)blockIdx.x * 32 + tx) * VEC;
  const bool active = c0 < cols;
  float acc[4][VEC];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[u][v] = 0.f;
  const long long stride = (long long)gridDim.y * 8;
  long long r = (long long)blockIdx.y * 8 + ty;
  if (active) {
    for (; r + 3 * stride < rows; r += 4 * stride) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float* p = x + (r + u * stride) * ld + c0;
        if constexpr (VEC == 4) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(p));
          acc[u][0] += v.x; acc[u][1] += v.y; acc[u][2] += v.z; acc[u][3] += v.w;
        } else {
          acc[u][0] += __ldg(p);
        }
      }
    }
    for (; r < rows; r += stride) {
      const float* p = x + r * ld + c0;
      if constexpr (VEC == 4) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(p));
        acc[0][0] += v.x; acc[0][1] += v.y; acc[0][2] += v.z; acc[0][3] += v.w;
      } else {
        acc[0][0] += __ldg(p);
      }
    }
  }
#pragma unroll
  for (int v = 0; v < VEC; ++v) red[ty][tx * VEC + v] = (acc[0][v] + acc[1][v]) + (acc[2][v] + acc[3][v]);
  __syncthreads();
  const int t = ty * 32 + tx;                       // 256 threads over the 32*VEC columns of the tile
  const long long tile0 = (long long)blockIdx.x * 32 * VEC;
  if (t < 32 * VEC && tile0 + t < cols) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += red[k][t];
    if (gridDim.y == 1) out[tile0 + t] = s;
    else part[(long long)blockIdx.y * cols + tile0 + t] = s;
  }
  if (gridDim.y == 1) return;
  __threadfence();
  __syncthreads();
  if (t == 0) last = (atomicAdd(&counters[blockIdx.x], 1u) == gridDim.y - 1);
  __syncthreads();
  if (!last) return;
  __threadfence();
  // final pass: the 8 row groups each add every 8th partial row (fixed order -> deterministic), then one smem reduce
  float fin[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) fin[v] = 0.f;
  if (active) {
    for (unsigned int k = ty; k < gridDim.y; k += 8) {
      const float* p = part + (long long)k * cols + c0;
      if constexpr (VEC == 4) {
        const float4 v = __ldcg(reinterpret_cast<const float4*>(p));
        fin[0] += v.x; fin[1] += v.y; fin[2] += v.z; fin[3] += v.w;
      } else {
        fin[0] += __ldcg(p);
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int v = 0; v < VEC; ++v) red[ty][tx * VEC + v] = fin[v];
  __syncthreads();
  if (t < 32 * VEC && tile0 + t < cols) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += red[k][t];
    out[tile0 + t] = s;
  }
  if (t == 0) counters[blockIdx.x] = 0u;
}

static void colsum_shape(long long rows, long long cols, int vec, long long& tiles, long long& splits) {
  tiles = (cols + 32 * vec - 1) / (32 * vec);
  splits = (132LL * 4) / tiles;                     // ~4 CTAs per SM in flight ...
  const long long max_splits = (rows + 63) / 64;    // ... each with at least 64 rows (8 per row group)
  if (splits > max_splits) splits = max_splits;
  if (splits > 256) splits = 256;                   // bounds the final pass (32 partial rows per row group)
  if (splits < 1) splits = 1;
}

// ------------------------------------------------------------------------------------------------ equivariant LayerNorm
// EquivariantLayerNormV2 ('component', nets/layer_norm.py:89-152) on e3nn-layout rows [N, sum mul*(2l+1)]:
// per entry: scalars are mean-centred over channels; n = mean over (channel, component) of field^2;
// out = field * (n + eps)^-1/2 * w[channel] (+ b[channel] on scalars).  One warp per node row; the eager version is
// ~35 tiny launches forward and ~70 backward per call (node-level tensors: pure launch overhead).
struct ELNArgs {
  const float* x; const float* w; const float* b;
  float* y; float* rstd;                       // rstd [N, n_entries]
  const float* gy; float* gx; float* dw_part; float* db_part;   // partial rows [grid, n_w] / [grid, n_b]
  int n_entries, dim, n_w, n_b;
  int mul[EQF_MAX_BLOCKS], d[EQF_MAX_BLOCKS], scalar[EQF_MAX_BLOCKS], off[EQF_MAX_BLOCKS], woff[EQF_MAX_BLOCKS], boff[EQF_MAX_BLOCKS];
  float eps; long long N;
  // planar variant: one packed [N, d, mul] buffer per entry (channel innermost) instead of e3nn-layout rows
  int planar;
  const float* xp[EQF_MAX_BLOCKS]; float* yp[EQF_MAX_BLOCKS]; const float* gyp[EQF_MAX_BLOCKS]; float* gxp[EQF_MAX_BLOCKS];
};

// entry t of row r: base pointer of its mul*d values, and the channel of the i-th value
__device__ __forceinline__ const float* eln_in(const ELNArgs& a, const float* rows, const float* const* blocks, long long r, int t) {
  return a.planar ? blocks[t] + r * (a.mul[t] * a.d[t]) : rows + r * a.dim + a.off[t];
}
__device__ __forceinline__ float* eln_out(const ELNArgs& a, float* rows, float* const* blocks, long long r, int t) {
  return a.planar ? blocks[t] + r * (a.mul[t] * a.d[t]) : rows + r * a.dim + a.off[t];
}
__device__ __forceinline__ int eln_chan(const ELNArgs& a, int t, int i) { return a.planar ? i % a.mul[t] : i / a.d[t]; }

__global__ void __launch_bounds__(256) eln_fwd_kernel(ELNArgs a) {
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = (long long)gridDim.x * 8;
  // one warp per (row, irreps entry): three times the parallelism of a warp per row on these latency-bound node tensors
  for (long long task = warp; task < a.N * a.n_entries; task += n_warps) {
    const long long r = task / a.n_entries;
    {
      const int t = (int)(task - r * a.n_entries);
      const int mul = a.mul[t], d = a.d[t], n = mul * d;
      const float* xe = eln_in(a, a.x, a.xp, r, t);
      float* ye = eln_out(a, a.y, a.yp, r, t);
      float mean = 0.f;
      if (a.scalar[t]) {
        float s = 0.f;
        for (int i = lane; i < n; i += 32) s += __ldg(xe + i);
        mean = wsum(s) / n;
      }
      float ss = 0.f;
      for (int i = lane; i < n; i += 32) { const float f = __ldg(xe + i) - mean; ss += f * f; }
      const float rs = rsqrtf(wsum(ss) / n + a.eps);
      for (int i = lane; i < n; i += 32) {
        const int c = eln_chan(a, t, i);
        float v = (__ldg(xe + i) - mean) * rs * __ldg(a.w + a.woff[t] + c);
        if (a.scalar[t]) v += __ldg(a.b + a.boff[t] + c);
        ye[i] = v;
      }
      if (lane == 0) a.rstd[r * a.n_entries + t] = rs;
    }
  }
}

__global__ void __launch_bounds__(256) eln_bwd_kernel(ELNArgs a) {
  extern __shared__ float sacc[];   // [n_w + n_b]
  for (int i = threadIdx.x; i < a.n_w + a.n_b; i += blockDim.x) sacc[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), n_warps = (long long)gridDim.x * 8;
  for (long long task = warp; task < a.N * a.n_entries; task += n_warps) {
    const long long r = task / a.n_entries;
    {
      const int t = (int)(task - r * a.n_entries);
      const int mul = a.mul[t], d = a.d[t], n = mul * d;
      const float* xe = eln_in(a, a.x, a.xp, r, t);
      const float* ge = eln_in(a, a.gy, a.gyp, r, t);
      float* gxe = eln_out(a, a.gx, a.gxp, r, t);
      const float rs = __ldg(a.rstd + r * a.n_entries + t);
      float mean = 0.f;
      if (a.scalar[t]) {
        float s = 0.f;
        for (int i = lane; i < n; i += 32) s += __ldg(xe + i);
        mean = wsum(s) / n;
      }
      // s1 = sum g*w*f
      float s1 = 0.f;
      for (int i = lane; i < n; i += 32) {
        const int c = eln_chan(a, t, i);
        const float f = __ldg(xe + i) - mean, g = __ldg(ge + i);
        s1 += g * __ldg(a.w + a.woff[t] + c) * f;
        atomicAdd(&sacc[a.woff[t] + c], g * f * rs);
        if (a.scalar[t]) atomicAdd(&sacc[a.n_w + a.boff[t] + c], g);
      }
      s1 = wsum(s1);
      const float k = -s1 * rs * rs * rs / n;           // dL/dn * 2/n with dL/dn = -1/2 r^3 s1
      float gsum = 0.f;
      for (int i = lane; i < n; i += 32) {
        const int c = eln_chan(a, t, i);
        const float f = __ldg(xe + i) - mean;
        const float gf = __ldg(ge + i) * rs * __ldg(a.w + a.woff[t] + c) + f * k;
        gxe[i] = gf;
        gsum += gf;
      }
      if (a.scalar[t]) {                                  // centring: g_x = g_f - mean(g_f)
        const float gm = wsum(gsum) / n;
        for (int i = lane; i < n; i += 32) gxe[i] -= gm;
      }
    }
  }
  __syncthreads();
  // one partial row per CTA: [d weight (n_w) | d bias (n_b)]
  for (int i = threadIdx.x; i < a.n_w + a.n_b; i += blockDim.x) a.dw_part[(long long)blockIdx.x * (a.n_w + a.n_b) + i] = sacc[i];
}

static int eln_grid(long long rows, int n_entries = 1) {
  long long blocks = (rows * n_entries + 7) / 8;
  if (blocks > 132LL * 4) blocks = 132LL * 4;
  return (int)(blocks < 1 ? 1 : blocks);
}

static int fill_eln(const EqfNormLayout* lay, ELNArgs& a) {
  if (lay == nullptr || lay->n_entries < 1 || lay->n_entries > EQF_MAX_BLOCKS) { set_error("bad norm layout"); return EQF_ERR_INVALID; }
  a.n_entries = lay->n_entries; a.eps = lay->eps;
  int off = 0, woff = 0, boff = 0;
  for (int t = 0; t < lay->n_entries; ++t) {
    if (lay->mul[t] < 1 || lay->d[t] < 1) { set_error("bad norm entry"); return EQF_ERR_INVALID; }
    a.mul[t] = lay->mul[t]; a.d[t] = lay->d[t]; a.scalar[t] = lay->is_scalar[t];
    a.off[t] = off; a.woff[t] = woff; a.boff[t] = boff;
    off += lay->mul[t] * lay->d[t]; woff += lay->mul[t];
    if (lay->is_scalar[t]) boff += lay->mul[t];
  }
  a.dim = off; a.n_w = woff; a.n_b = boff;
  a.planar = 0;
  return EQF_OK;
}

static int pointwise_grid(long long rows) {
  long long blocks = (rows + 7) / 8;
  const long long cap = 132LL * 8;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

}  // namespace eqf

using namespace eqf;

extern "C" int eqf_pointwise_rows(int64_t rows) { return pointwise_grid(rows); }

extern "C" int eqf_ln_silu_fwd(const float* x, const float* bias, const float* gamma, const float* beta, float eps,
                               int64_t R, int32_t C, float* y, float* mean, float* rstd, void* stream) {
  if (R == 0) return EQF_OK;
  if (!x || !gamma || !beta || !y || !mean || !rstd) { set_error("eqf_ln_silu_fwd: null pointer"); return EQF_ERR_INVALID; }
  if (C < 1 || C > 32 * kMaxPerLane) { set_error("eqf_ln_silu: C must be in 1..256"); return EQF_ERR_UNSUPPORTED; }
  cudaStream_t st = (cudaStream_t)stream;
  const bool al16 = ((((uintptr_t)x | (uintptr_t)y | (uintptr_t)gamma | (uintptr_t)beta | (uintptr_t)bias) & 15) == 0);
  if (C == 64 && al16) ln_silu_fwd64_kernel<<<pointwise_grid((R + 1) / 2), 256, 0, st>>>(x, bias, gamma, beta, eps, R, y, mean, rstd);
  else if (C <= 64) ln_silu_fwd_kernel<2><<<pointwise_grid(R), 256, 0, st>>>(x, bias, gamma, beta, eps, R, C, y, mean, rstd);
  else if (C <= 128) ln_silu_fwd_kernel<4><<<pointwise_grid(R), 256, 0, st>>>(x, bias, gamma, beta, eps, R, C, y, mean, rstd);
  else ln_silu_fwd_kernel<8><<<pointwise_grid(R), 256, 0, st>>>(x, bias, gamma, beta, eps, R, C, y, mean, rstd);
  return check_cuda(cudaGetLastError(), "ln_silu_fwd_kernel launch");
}

extern "C" int eqf_ln_silu_bwd(const float* x, const float* bias, const float* gamma, const float* beta, const float* mean,
                               const float* rstd, const float* gy, int64_t R, int32_t C, float* gx, float* part,
                               void* stream) {
  if (R == 0) return EQF_OK;
  if (!x || !gamma || !beta || !mean || !rstd || !gy || !gx || !part) {
    set_error("eqf_ln_silu_bwd: null pointer"); return EQF_ERR_INVALID;
  }
  if (C < 1 || C > 32 * kMaxPerLane) { set_error("eqf_ln_silu: C must be in 1..256"); return EQF_ERR_UNSUPPORTED; }
  cudaStream_t st = (cudaStream_t)stream;
  const bool al16 = ((((uintptr_t)x | (uintptr_t)gx | (uintptr_t)gy | (uintptr_t)gamma | (uintptr_t)beta | (uintptr_t)bias) & 15) == 0);
  // NB: the partial buffer always has eqf_pointwise_rows(R) rows; the 64-wide kernel launches that many CTAs as well
  if (C == 64 && al16) ln_silu_bwd64_kernel<<<pointwise_grid(R), 256, 0, st>>>(x, bias, gamma, beta, mean, rstd, gy, R, gx, part);
  else if (C <= 64) ln_silu_bwd_kernel<2><<<pointwise_grid(R), 256, 0, st>>>(x, bias, gamma, beta, mean, rstd, gy, R, C, gx, part);
  else if (C <= 128) ln_silu_bwd_kernel<4><<<pointwise_grid(R), 256, 0, st>>>(x, bias, gamma, beta, mean, rstd, gy, R, C, gx, part);
  else ln_silu_bwd_kernel<8><<<pointwise_grid(R), 256, 0, st>>>(x, bias, gamma, beta, mean, rstd, gy, R, C, gx, part);
  return check_cuda(cudaGetLastError(), "ln_silu_bwd_kernel launch");
}

static int fill_gate(const EqfGateLayout* lay, GateArgs& a) {
  if (lay == nullptr) { set_error("null gate layout"); return EQF_ERR_INVALID; }
  if (lay->n_gated < 0 || lay->n_gated > EQF_MAX_BLOCKS || lay->n_heads < 1 || lay->n_alpha % lay->n_heads != 0) {
    set_error("bad gate layout"); return EQF_ERR_INVALID;
  }
  a.n_gated = lay->n_gated; a.A0 = lay->n_alpha; a.S = lay->n_scalars; a.H = lay->n_heads;
  a.Gt = 0;
  for (int b = 0; b < lay->n_gated; ++b) { a.d[b] = lay->d[b]; a.C[b] = lay->C[b]; a.Gt += lay->C[b]; }
  a.c_silu = lay->c_silu; a.c_sig = lay->c_sigmoid; a.c_slr = lay->c_slr; a.slope = lay->slr_slope;
  return EQF_OK;
}

extern "C" int eqf_gate_logits_fwd(const EqfGateLayout* lay, const float* t0, const float* bias,
                                   const float* const* gated, const float* alpha_dot, int64_t n_edges, float* z,
                                   float* v0, float* const* vout, void* stream) {
  GateArgs a;
  int rc = fill_gate(lay, a);
  if (rc != EQF_OK || n_edges == 0) return rc;
  if (!t0 || !alpha_dot || !z || !v0) { set_error("eqf_gate_logits_fwd: null pointer"); return EQF_ERR_INVALID; }
  a.t0 = t0; a.bias = bias; a.alpha_dot = alpha_dot; a.z = z; a.v0 = v0; a.E = n_edges;
  for (int b = 0; b < a.n_gated; ++b) {
    if (!gated || !vout || !gated[b] || !vout[b]) { set_error("eqf_gate_logits_fwd: null block"); return EQF_ERR_INVALID; }
    a.gated[b] = gated[b]; a.vout[b] = vout[b];
  }
  if (gate_vec_ok(a)) gate_logits_fwd_vec_kernel<<<pointwise_grid(n_edges), 256, 0, (cudaStream_t)stream>>>(a);
  else gate_logits_fwd_kernel<<<pointwise_grid(n_edges), 256, 0, (cudaStream_t)stream>>>(a);
  return check_cuda(cudaGetLastError(), "gate_logits_fwd_kernel launch");
}

extern "C" int eqf_gate_logits_bwd(const EqfGateLayout* lay, const float* t0, const float* bias,
                                   const float* const* gated, const float* alpha_dot, const float* gz, const float* gv0,
                                   const float* const* gvout, int64_t n_edges, float* gt0, float* const* ggated,
                                   float* gdot_part, void* stream) {
  GateArgs a;
  int rc = fill_gate(lay, a);
  if (rc != EQF_OK || n_edges == 0) return rc;
  if (!t0 || !alpha_dot || !gz || !gv0 || !gt0 || !gdot_part) { set_error("eqf_gate_logits_bwd: null pointer"); return EQF_ERR_INVALID; }
  a.t0 = t0; a.bias = bias; a.alpha_dot = alpha_dot; a.gz = gz; a.gv0 = gv0; a.gt0 = gt0; a.gdot_part = gdot_part; a.E = n_edges;
  for (int b = 0; b < a.n_gated; ++b) {
    if (!gated || !gvout || !ggated || !gated[b] || !gvout[b] || !ggated[b]) { set_error("eqf_gate_logits_bwd: null block"); return EQF_ERR_INVALID; }
    a.gated[b] = gated[b]; a.gvout[b] = gvout[b]; a.ggated[b] = ggated[b];
  }
  if (gate_vec_ok(a)) gate_logits_bwd_vec_kernel<<<pointwise_grid(n_edges), 256, a.A0 * sizeof(float), (cudaStream_t)stream>>>(a);
  else gate_logits_bwd_kernel<<<pointwise_grid(n_edges), 256, a.A0 * sizeof(float), (cudaStream_t)stream>>>(a);
  return check_cuda(cudaGetLastError(), "gate_logits_bwd_kernel launch");
}


extern "C" int eqf_eln_rows(const EqfNormLayout* lay, int64_t rows) { return eln_grid(rows, lay ? lay->n_entries : 1); }

extern "C" int eqf_eln_fwd(const EqfNormLayout* lay, const float* x, const float* w, const float* b, int64_t N, float* y,
                           float* rstd, void* stream) {
  ELNArgs a;
  int rc = fill_eln(lay, a);
  if (rc != EQF_OK || N == 0) return rc;
  if (!x || !w || !y || !rstd || (a.n_b > 0 && !b)) { set_error("eqf_eln_fwd: null pointer"); return EQF_ERR_INVALID; }
  a.x = x; a.w = w; a.b = b; a.y = y; a.rstd = rstd; a.N = N;
  eln_fwd_kernel<<<eln_grid(N, a.n_entries), 256, 0, (cudaStream_t)stream>>>(a);
  return check_cuda(cudaGetLastError(), "eln_fwd_kernel launch");
}

extern "C" int eqf_eln_bwd(const EqfNormLayout* lay, const float* x, const float* w, const float* rstd, const float* gy,
                           int64_t N, float* gx, float* part, void* stream) {
  ELNArgs a;
  int rc = fill_eln(lay, a);
  if (rc != EQF_OK || N == 0) return rc;
  if (!x || !w || !rstd || !gy || !gx || !part) { set_error("eqf_eln_bwd: null pointer"); return EQF_ERR_INVALID; }
  a.x = x; a.w = w; a.b = nullptr; a.rstd = const_cast<float*>(rstd); a.gy = gy; a.gx = gx; a.dw_part = part; a.db_part = nullptr; a.N = N;
  eln_bwd_kernel<<<eln_grid(N, a.n_entries), 256, (a.n_w + a.n_b) * sizeof(float), (cudaStream_t)stream>>>(a);
  return check_cuda(cudaGetLastError(), "eln_bwd_kernel launch");
}


// out[cols] = column sums of x[rows, cols] (row stride ld).  `part` needs eqf_colsum_scratch_floats(rows, cols) floats,
// `counters` EQF_COLSUM_COUNTERS zero-initialised uint32 (left zeroed on return: reusable across calls on one stream).
extern "C" int64_t eqf_colsum_scratch_floats(int64_t rows, int64_t cols) {
  long long tiles, splits;
  colsum_shape(rows, cols, 1, tiles, splits);       // the scalar layout has the most tiles -> fewest splits; bound both
  long long t4, s4;
  colsum_shape(rows, cols, 4, t4, s4);
  const long long m = splits > s4 ? splits : s4;
  return m * cols;
}

extern "C" int eqf_colsum(const float* x, int64_t rows, int64_t cols, int64_t ld, float* out, float* part,
                          uint32_t* counters, void* stream) {
  if (cols <= 0) return EQF_OK;
  if (!out) { set_error("eqf_colsum: null output"); return EQF_ERR_INVALID; }
  cudaStream_t s = (cudaStream_t)stream;
  if (rows <= 0) return check_cuda(cudaMemsetAsync(out, 0, cols * sizeof(float), s), "eqf_colsum memset");
  if (!x || !part || !counters || ld < cols) { set_error("eqf_colsum: bad arguments"); return EQF_ERR_INVALID; }
  const bool vec = (cols % 4 == 0) && (ld % 4 == 0) && ((uintptr_t)x % 16 == 0);
  long long tiles, splits;
  colsum_shape(rows, cols, vec ? 4 : 1, tiles, splits);
  if (tiles > EQF_COLSUM_COUNTERS) { set_error("eqf_colsum: too many column tiles"); return EQF_ERR_UNSUPPORTED; }
  dim3 grid((unsigned)tiles, (unsigned)splits), block(32, 8);
  if (vec) colsum_kernel<4><<<grid, block, 0, s>>>(x, rows, cols, ld, out, part, counters);
  else colsum_kernel<1><<<grid, block, 0, s>>>(x, rows, cols, ld, out, part, counters);
  return check_cuda(cudaGetLastError(), "colsum_kernel launch");
}


// planar variants: entry t of the node features is a packed [N, d_t, mul_t] buffer (channel innermost), as the GEMM /
// tensor-product kernels keep them - the transformer blocks then never leave the planar layout
extern "C" int eqf_eln_fwd_planar(const EqfNormLayout* lay, const float* const* x_blocks, const float* w, const float* b,
                                  int64_t N, float* const* y_blocks, float* rstd, void* stream) {
  ELNArgs a;
  int rc = fill_eln(lay, a);
  if (rc != EQF_OK || N == 0) return rc;
  if (!x_blocks || !y_blocks || !w || !rstd || (a.n_b > 0 && !b)) { set_error("eqf_eln_fwd_planar: null pointer"); return EQF_ERR_INVALID; }
  a.planar = 1; a.x = nullptr; a.y = nullptr; a.w = w; a.b = b; a.rstd = rstd; a.N = N;
  for (int t = 0; t < a.n_entries; ++t) {
    if (!x_blocks[t] || !y_blocks[t]) { set_error("eqf_eln_fwd_planar: null block"); return EQF_ERR_INVALID; }
    a.xp[t] = x_blocks[t]; a.yp[t] = y_blocks[t];
  }
  eln_fwd_kernel<<<eln_grid(N, a.n_entries), 256, 0, (cudaStream_t)stream>>>(a);
  return check_cuda(cudaGetLastError(), "eln_fwd_kernel (planar) launch");
}

extern "C" int eqf_eln_bwd_planar(const EqfNormLayout* lay, const float* const* x_blocks, const float* w, const float* rstd,
                                  const float* const* gy_blocks, int64_t N, float* const* gx_blocks, float* part,
                                  void* stream) {
  ELNArgs a;
  int rc = fill_eln(lay, a);
  if (rc != EQF_OK || N == 0) return rc;
  if (!x_blocks || !gy_blocks || !gx_blocks || !w || !rstd || !part) { set_error("eqf_eln_bwd_planar: null pointer"); return EQF_ERR_INVALID; }
  a.planar = 1; a.x = nullptr; a.gy = nullptr; a.gx = nullptr; a.w = w; a.b = nullptr; a.rstd = const_cast<float*>(rstd);
  a.dw_part = part; a.db_part = nullptr; a.N = N;
  for (int t = 0; t < a.n_entries; ++t) {
    if (!x_blocks[t] || !gy_blocks[t] || !gx_blocks[t]) { set_error("eqf_eln_bwd_planar: null block"); return EQF_ERR_INVALID; }
    a.xp[t] = x_blocks[t]; a.gyp[t] = gy_blocks[t]; a.gxp[t] = gx_blocks[t];
  }
  eln_bwd_kernel<<<eln_grid(N, a.n_entries), 256, (a.n_w + a.n_b) * sizeof(float), (cudaStream_t)stream>>>(a);
  return check_cuda(cudaGetLastError(), "eln_bwd_kernel (planar) launch");
}


// Gaussian radial basis with K = 128 functions (gaussian_rbf.py:5-40): out [E, 128]
extern "C" int eqf_rbf_fwd(const float* dist, const float* mean, const float* std, const float* weight, const float* bias,
                           float cutoff, int64_t n_edges, float* out, void* stream) {
  if (n_edges == 0) return EQF_OK;
  if (!dist || !mean || !std || !weight || !bias || !out || cutoff == 0.f) { set_error("eqf_rbf_fwd: bad arguments"); return EQF_ERR_INVALID; }
  rbf_fwd_kernel<<<pointwise_grid(n_edges), 256, 0, (cudaStream_t)stream>>>(dist, mean, std, weight, bias, 1.f / cutoff, n_edges, out);
  return check_cuda(cudaGetLastError(), "rbf_fwd_kernel launch");
}

// g_dist [E] and partial rows part[eqf_pointwise_rows(E)][258] = d mean | d std | d weight | d bias
extern "C" int eqf_rbf_bwd(const float* dist, const float* mean, const float* std, const float* weight, const float* bias,
                           float cutoff, const float* g, int64_t n_edges, float* g_dist, float* part, void* stream) {
  if (n_edges == 0) return EQF_OK;
  if (!dist || !mean || !std || !weight || !bias || !g || !g_dist || !part || cutoff == 0.f) { set_error("eqf_rbf_bwd: bad arguments"); return EQF_ERR_INVALID; }
  rbf_bwd_kernel<<<pointwise_grid(n_edges), 256, 0, (cudaStream_t)stream>>>(dist, mean, std, weight, bias, 1.f / cutoff, g, n_edges,
                                                                             g_dist, part);
  return check_cuda(cudaGetLastError(), "rbf_bwd_kernel launch");
}
