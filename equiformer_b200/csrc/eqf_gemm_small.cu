// eqf_gemm_small.cu - grouped fp32 GEMM for the SMALL products of the path (sm_90a, CUDA cores, exact fp32 FMA).
//
// Node-level linears (nets/graph_attention_transformer.py:430-431 merge_src / merge_dst, :515 proj, the FeedForwardNetwork's
// two FCTPs, nets/tensor_product_rescale.py LinearRS) are one [atoms * (2l+1), mul_in] x [mul_in, mul_out] product per degree:
// 2 324 atoms x {1, 3, 5} rows against 128 / 64 / 32 channels - 30 to 80 MFLOP each: one cuBLAS call per degree would
// mean ~180 small launches per step, and the wgmma kernels need M >= 16 k rows to pay for their prologue.  Here ONE launch carries all degrees of a linear (and, in the backward, the data gradients AND the weight
// gradients of all degrees): a table of up to EQF_GROUP_MAX problems
//     C_i[M, N] (+)= alpha_i * sum_k A_i(m, k) B_i(k, n)
// whose operands are addressed through (contiguous-along-k | contiguous-along-m/n) flags, so the same tile code serves
//     forward        x[M, K] W[K, N]            A k-contiguous, B n-contiguous
//     data gradient  g[M, N'] W[K', N']^T       A k-contiguous, B k-contiguous
//     weight grad.   x[R, K']^T g[R, N]         A m-contiguous, B n-contiguous, the long reduction over R split across CTAs
//                                               (fp32 atomic adds into a zeroed output, like the reference's scatter)
// 64 x 64 output tile per CTA, 256 threads x (4 x 4) accumulators, 16-deep k-chunks double-buffered in shared memory,
// 128-bit global loads along the contiguous dimension.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdlib>
#include <string>

#include "eqf_common.cuh"

namespace eqf {
namespace small {

constexpr int BM = 64, BN = 64, BK = 16, kThreadsG = 256, kPad = 4;

struct Prob {
  const float* A;
  const float* B;
  float* C;
  int M, N, K;
  int lda, ldb, ldc;
  int a_kc, b_kc;          // 1: contiguous along k
  float alpha;
  int tiles_m, tiles_n, splits, k_per_split;
  int atomic;              // add into C with fp32 atomics (split reduction) instead of storing
  int tile0;               // first CTA of the problem
};
struct Args {
  int n;
  Prob p[EQF_GROUP_MAX];
};

template <bool AKC, bool BKC>
__device__ __forceinline__ void load_tiles(const Prob& p, int m0, int n0, int k0, int k_end, float4& ra, float4& rb) {
  const int t = threadIdx.x;
  ra = make_float4(0.f, 0.f, 0.f, 0.f);
  rb = make_float4(0.f, 0.f, 0.f, 0.f);
  if constexpr (AKC) {           // A[m * lda + k]: thread = (row t / 4, k-quad t % 4)
    const int m = m0 + (t >> 2), k = k0 + (t & 3) * 4;
    if (m < p.M && k < k_end) ra = __ldg(reinterpret_cast<const float4*>(p.A + (size_t)m * p.lda + k));
  } else {                       // A[k * lda + m]: thread = (k t / 16, m-quad t % 16)
    const int k = k0 + (t >> 4), m = m0 + (t & 15) * 4;
    if (k < k_end && m < p.M) ra = __ldg(reinterpret_cast<const float4*>(p.A + (size_t)k * p.lda + m));
  }
  if constexpr (BKC) {           // B[n * ldb + k]
    const int n = n0 + (t >> 2), k = k0 + (t & 3) * 4;
    if (n < p.N && k < k_end) rb = __ldg(reinterpret_cast<const float4*>(p.B + (size_t)n * p.ldb + k));
  } else {                       // B[k * ldb + n]
    const int k = k0 + (t >> 4), n = n0 + (t & 15) * 4;
    if (k < k_end && n < p.N) rb = __ldg(reinterpret_cast<const float4*>(p.B + (size_t)k * p.ldb + n));
  }
}

template <bool AKC, bool BKC>
__device__ __forceinline__ void store_tiles(float (*As)[BM + kPad], float (*Bs)[BN + kPad], const float4& ra, const float4& rb) {
  const int t = threadIdx.x;
  if constexpr (AKC) {
    const int m = t >> 2, k = (t & 3) * 4;
    As[k][m] = ra.x; As[k + 1][m] = ra.y; As[k + 2][m] = ra.z; As[k + 3][m] = ra.w;
  } else {
    *reinterpret_cast<float4*>(&As[t >> 4][(t & 15) * 4]) = ra;
  }
  if constexpr (BKC) {
    const int n = t >> 2, k = (t & 3) * 4;
    Bs[k][n] = rb.x; Bs[k + 1][n] = rb.y; Bs[k + 2][n] = rb.z; Bs[k + 3][n] = rb.w;
  } else {
    *reinterpret_cast<float4*>(&Bs[t >> 4][(t & 15) * 4]) = rb;
  }
}

template <bool AKC, bool BKC>
__device__ __forceinline__ void tile(const Prob& p, int tm, int tn, int split, float (*As)[BK][BM + kPad], float (*Bs)[BK][BN + kPad]) {
  const int m0 = tm * BM, n0 = tn * BN;
  const int k_begin = split * p.k_per_split;
  const int k_end = (k_begin + p.k_per_split) < p.K ? (k_begin + p.k_per_split) : p.K;
  const int t = threadIdx.x, ty = t >> 4, tx = t & 15;      // rows 4 ty .., columns 4 tx ..
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float4 ra, rb;
  load_tiles<AKC, BKC>(p, m0, n0, k_begin, k_end, ra, rb);
  store_tiles<AKC, BKC>(As[0], Bs[0], ra, rb);
  __syncthreads();
  int buf = 0;
  for (int k0 = k_begin; k0 < k_end; k0 += BK) {
    const bool more = (k0 + BK) < k_end;
    if (more) load_tiles<AKC, BKC>(p, m0, n0, k0 + BK, k_end, ra, rb);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (more) {
      store_tiles<AKC, BKC>(As[buf ^ 1], Bs[buf ^ 1], ra, rb);
      __syncthreads();
      buf ^= 1;
    }
  }
  const int n = n0 + tx * 4;
  if (n >= p.N) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= p.M) break;
    float* c = p.C + (size_t)m * p.ldc + n;
    if (!p.atomic) {
      *reinterpret_cast<float4*>(c) = make_float4(p.alpha * acc[i][0], p.alpha * acc[i][1], p.alpha * acc[i][2], p.alpha * acc[i][3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) atomicAdd(c + j, p.alpha * acc[i][j]);
    }
  }
}

__global__ void __launch_bounds__(kThreadsG) grouped_gemm_kernel(const __grid_constant__ Args g) {
  __shared__ __align__(16) float As[2][BK][BM + kPad];
  __shared__ __align__(16) float Bs[2][BK][BN + kPad];
  int pi = 0;
  for (int i = 1; i < g.n; ++i) if ((int)blockIdx.x >= g.p[i].tile0) pi = i;
  const Prob& p = g.p[pi];
  int local = (int)blockIdx.x - p.tile0;
  const int tn = local % p.tiles_n; local /= p.tiles_n;
  const int tm = local % p.tiles_m;
  const int split = local / p.tiles_m;
  if (p.a_kc) {
    if (p.b_kc) tile<true, true>(p, tm, tn, split, As, Bs);
    else tile<true, false>(p, tm, tn, split, As, Bs);
  } else {
    if (p.b_kc) tile<false, true>(p, tm, tn, split, As, Bs);
    else tile<false, false>(p, tm, tn, split, As, Bs);
  }
}

// ---------------------------------------------------------------------------------------------- warp-MMA variant
// The same tiles on the tensor cores' warp-level path (mma.sync m16n8k8, tf32 inputs, fp32 accumulate) with the 3xTF32
// split done in registers: a = a_hi + a_lo, b = b_hi + b_lo, acc += a_lo b_hi + a_hi b_lo + a_hi b_hi (the error of the
// dropped a_lo b_lo term is ~2^-22 relative, like the wgmma kernels of eqf_gemm_tf32x3.cu).  The CUDA-core kernel
// above is bound by FMA issue (a 64 x 64 x 128 tile is 16 k warp-FMAs); here a k-step of 8 costs a
// warp 24 MMAs + 16 shared loads + 48 split instructions for its 32 x 32 sub-tile instead of 256 FMAs + 32 loads.
// 128 threads = 4 warps (2 x 2) per 64 x 64 tile; operands in shared memory in whichever orientation makes the global
// load a 128-bit access AND the fragment loads conflict-free: k-contiguous operands as [row][16 + 4], the others as
// [k][64 + 8].
constexpr int kThreadsM = 128, kLdK = BK + 4, kLdN = 64 + 8, kMmaStages = 4;
constexpr int kTileFloats = (64 * kLdK) > (BK * kLdN) ? (64 * kLdK) : (BK * kLdN);

__device__ __forceinline__ float rn_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u); }

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// 64 x 16 (or 16 x 64) operand tile: two 16-byte cp.async per thread along the contiguous dimension, straight into the
// shared-memory orientation the fragments are read from (out-of-range pieces are zero-filled: src-size 0)
template <bool KC>
__device__ __forceinline__ void mma_load_async(float* sm, const float* base, int ld, int rows, int r0, int k0, int k_end) {
  const int t = threadIdx.x;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int i = t + h * kThreadsM;
    const float* src;
    float* dst;
    bool ok;
    if constexpr (KC) {          // base[r * ld + k]
      const int r = r0 + (i >> 2), k = k0 + (i & 3) * 4;
      ok = r < rows && k < k_end;
      src = base + (size_t)(ok ? r : 0) * ld + (ok ? k : 0);
      dst = sm + (i >> 2) * kLdK + (i & 3) * 4;
    } else {                     // base[k * ld + r]
      const int k = k0 + (i >> 4), r = r0 + (i & 15) * 4;
      ok = k < k_end && r < rows;
      src = base + (size_t)(ok ? k : 0) * ld + (ok ? r : 0);
      dst = sm + (i >> 4) * kLdN + (i & 15) * 4;
    }
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src), "r"(ok ? 16 : 0) : "memory");
  }
}
template <bool KC>
__device__ __forceinline__ float mma_at(const float* sm, int r, int k) { return KC ? sm[r * kLdK + k] : sm[k * kLdN + r]; }

template <bool AKC, bool BKC>
__device__ __forceinline__ void mma_tile(const Prob& p, int tm, int tn, int split, float (*As)[kTileFloats], float (*Bs)[kTileFloats]) {
  const int m0 = tm * BM, n0 = tn * BN;
  const int k_begin = split * p.k_per_split;
  const int k_end = (k_begin + p.k_per_split) < p.K ? (k_begin + p.k_per_split) : p.K;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[i][j][c] = 0.f;
  // kMmaStages-deep cp.async ring: with one chunk of register prefetch every 16-deep chunk costs a full L2 round trip
  const int n_chunks = (k_end - k_begin + BK - 1) / BK;
#pragma unroll
  for (int s = 0; s < kMmaStages - 1; ++s) {
    if (s < n_chunks) {
      mma_load_async<AKC>(As[s], p.A, p.lda, p.M, m0, k_begin + s * BK, k_end);
      mma_load_async<BKC>(Bs[s], p.B, p.ldb, p.N, n0, k_begin + s * BK, k_end);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  for (int c = 0; c < n_chunks; ++c) {
    asm volatile("cp.async.wait_group %0;" ::"n"(kMmaStages - 2) : "memory");
    __syncthreads();                       // chunk c landed for every thread; everyone is done with chunk c - 1's buffer
    {
      const int nc = c + kMmaStages - 1;
      if (nc < n_chunks) {
        mma_load_async<AKC>(As[nc % kMmaStages], p.A, p.lda, p.M, m0, k_begin + nc * BK, k_end);
        mma_load_async<BKC>(Bs[nc % kMmaStages], p.B, p.ldb, p.N, n0, k_begin + nc * BK, k_end);
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
    const int buf = c % kMmaStages;
#pragma unroll
    for (int ks = 0; ks < BK; ks += 8) {
      uint32_t ahi[2][4], alo[2][4], bhi[4][2], blo[4][2];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const int r = wm + mi * 16 + g;
        const float v[4] = {mma_at<AKC>(As[buf], r, ks + t), mma_at<AKC>(As[buf], r + 8, ks + t),
                            mma_at<AKC>(As[buf], r, ks + t + 4), mma_at<AKC>(As[buf], r + 8, ks + t + 4)};
#pragma unroll
        for (int cc = 0; cc < 4; ++cc) {
          const float h = rn_tf32(v[cc]);
          ahi[mi][cc] = __float_as_uint(h);
          alo[mi][cc] = __float_as_uint(v[cc] - h);
        }
      }
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const int n = wn + ni * 8 + g;
        const float v[2] = {mma_at<BKC>(Bs[buf], n, ks + t), mma_at<BKC>(Bs[buf], n, ks + t + 4)};
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
          const float h = rn_tf32(v[cc]);
          bhi[ni][cc] = __float_as_uint(h);
          blo[ni][cc] = __float_as_uint(v[cc] - h);
        }
      }
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
          mma_tf32(acc[mi][ni], alo[mi], bhi[ni]);
          mma_tf32(acc[mi][ni], ahi[mi], blo[ni]);
          mma_tf32(acc[mi][ni], ahi[mi], bhi[ni]);
        }
    }
  }
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni) {
      const int n = n0 + wn + ni * 8 + 2 * t;
      if (n >= p.N) continue;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int m = m0 + wm + mi * 16 + g + hh * 8;
        if (m >= p.M) continue;
        float* c = p.C + (size_t)m * p.ldc + n;
        const float v0 = p.alpha * acc[mi][ni][2 * hh], v1 = p.alpha * acc[mi][ni][2 * hh + 1];
        if (!p.atomic) *reinterpret_cast<float2*>(c) = make_float2(v0, v1);
        else { atomicAdd(c, v0); atomicAdd(c + 1, v1); }
      }
    }
}

__global__ void __launch_bounds__(kThreadsM) grouped_gemm_mma_kernel(const __grid_constant__ Args g) {
  __shared__ __align__(16) float As[kMmaStages][kTileFloats];
  __shared__ __align__(16) float Bs[kMmaStages][kTileFloats];
  int pi = 0;
  for (int i = 1; i < g.n; ++i) if ((int)blockIdx.x >= g.p[i].tile0) pi = i;
  const Prob& p = g.p[pi];
  int local = (int)blockIdx.x - p.tile0;
  const int tn = local % p.tiles_n; local /= p.tiles_n;
  const int tm = local % p.tiles_m;
  const int split = local / p.tiles_m;
  if (p.a_kc) {
    if (p.b_kc) mma_tile<true, true>(p, tm, tn, split, As, Bs);
    else mma_tile<true, false>(p, tm, tn, split, As, Bs);
  } else {
    if (p.b_kc) mma_tile<false, true>(p, tm, tn, split, As, Bs);
    else mma_tile<false, false>(p, tm, tn, split, As, Bs);
  }
}

}  // namespace small
}  // namespace eqf

using namespace eqf;

// n (<= EQF_GROUP_MAX) independent products in one launch.  Problem i:  C[M, N] = alpha * op(A) op(B)  with
//   mode 0: A[M, K] (lda) x B[K, N] (ldb);   mode 1: A[M, K] x B[N, K]^T;   mode 2: A[K, M]^T x B[K, N]   (gemm_raw's modes)
// fp32 FMA accumulation.  `accumulate` != 0: the reduction is split across CTAs and ADDED into C with fp32 atomics (C must
// hold the initial value, normally zero; used for the long reductions of the weight gradients); 0: C is overwritten.
// Pointers 16-byte aligned, leading dimensions and the extent of every contiguous dimension multiples of 4.
extern "C" int eqf_gemm_grouped(const EqfGemmProblem* problems, int32_t n, void* stream) {
  using namespace eqf::small;
  if (n <= 0) return EQF_OK;
  if (problems == nullptr || n > EQF_GROUP_MAX) { set_error("eqf_gemm_grouped: bad problem table"); return EQF_ERR_INVALID; }
  Args g;
  g.n = 0;
  int tiles = 0;
  int sms = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  for (int i = 0; i < n; ++i) {
    const EqfGemmProblem& q = problems[i];
    if (q.M <= 0 || q.N <= 0 || q.K <= 0) continue;
    if (!q.A || !q.B || !q.C || q.mode < 0 || q.mode > 2) { set_error("eqf_gemm_grouped: null pointer / bad mode"); return EQF_ERR_INVALID; }
    Prob& p = g.p[g.n];
    p.A = q.A; p.B = q.B; p.C = q.C;
    p.M = (int)q.M; p.N = (int)q.N; p.K = (int)q.K;
    p.lda = (int)q.lda; p.ldb = (int)q.ldb; p.ldc = (int)q.ldc;
    p.a_kc = q.mode != 2;          // modes 0, 1: A[M, K] row-major; mode 2: A[K, M]
    p.b_kc = q.mode == 1;          // mode 1: B[N, K]; modes 0, 2: B[K, N]
    p.alpha = q.alpha;
    const bool a_ok = p.a_kc ? (p.K % 4 == 0) : (p.M % 4 == 0);
    const bool b_ok = p.b_kc ? (p.K % 4 == 0) : (p.N % 4 == 0);
    if (!a_ok || !b_ok || p.N % 4 != 0 || ((p.lda | p.ldb | p.ldc) & 3) ||
        (((uintptr_t)q.A | (uintptr_t)q.B | (uintptr_t)q.C) & 15)) {
      set_error("eqf_gemm_grouped: operands must be 16-byte aligned with contiguous extents / leading dimensions % 4 == 0");
      return EQF_ERR_INVALID;
    }
    p.tiles_m = (p.M + BM - 1) / BM;
    p.tiles_n = (p.N + BN - 1) / BN;
    p.splits = 1;
    p.k_per_split = p.K;
    p.atomic = q.accumulate ? 1 : 0;
    if (q.accumulate) {            // aim at ~2 CTAs per SM over the whole reduction, at least 256 rows per slice
      const int out_tiles = p.tiles_m * p.tiles_n;
      int want = (2 * sms + out_tiles - 1) / out_tiles;
      const int max_splits = (p.K + 255) / 256;
      if (want > max_splits) want = max_splits;
      if (want < 1) want = 1;
      int per = (p.K + want - 1) / want;
      per = (per + BK - 1) / BK * BK;
      p.k_per_split = per;
      p.splits = (p.K + per - 1) / per;
    }
    p.tile0 = tiles;
    tiles += p.tiles_m * p.tiles_n * p.splits;
    ++g.n;
  }
  if (g.n == 0) return EQF_OK;
  // EQF_SMALL_MMA=0: the CUDA-core (exact fp32 FMA) kernel instead of the warp-MMA 3xTF32 one
  static const bool use_mma = [] { const char* e = std::getenv("EQF_SMALL_MMA"); return e == nullptr || e[0] != '0'; }();
  if (use_mma) small::grouped_gemm_mma_kernel<<<tiles, kThreadsM, 0, (cudaStream_t)stream>>>(g);
  else small::grouped_gemm_kernel<<<tiles, kThreadsG, 0, (cudaStream_t)stream>>>(g);
  return check_cuda(cudaGetLastError(), "grouped_gemm_kernel launch");
}
