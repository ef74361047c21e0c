// eqf_dtp_v3.cu - third-generation DTP kernels (sm_90a): software-pipelined tiles, one barrier per tile.
//
// What profiling of the second generation showed: DRAM traffic == algorithmic bytes but far from DRAM peak; FFMA a small
// share of the issued instructions (integer address/divide overhead), barrier + long-scoreboard stalls exposed because a tile went load-y -> barrier -> fold -> barrier -> work.
// This generation therefore
//   * pipelines the per-tile staging: edge harmonics of tile t+2 are loaded into registers while tile t is processed,
//     the fold M_p = C_p.y of tile t+1 runs before the work of tile t, buffers are double - ONE __syncthreads per tile;
//   * streams the per-edge radial weights AND (when not gathered) the in1 rows of the next tile with cp.async.bulk
//     (TMA, one mbarrier per stage) so the compute warps never wait on those loads;
//   * backward: one balanced (path x edge-group) task list like the forward - the in1-gradient is accumulated in a
//     double-buffered shared-memory tile with RED.shared and written out coalesced one tile later, the weight
//     gradient goes straight to HBM (or to a per-CTA shared accumulator for shared weights);
//   * power-of-two lane maps (shift/mask) and division-free staging loops.
#include <mutex>
#include <unordered_map>

#include "eqf_common.cuh"

namespace eqf {

struct S3 {
  const PathDev* paths;
  const float* cg;
  const int* mdesc;
  const int2* vwtasks;
  float* M[2];
  float* ysh[2];
  float* wacc;      // [w_numel]   shared-weight gradient accumulator (backward)
  float* gxacc[2];  // [te][d_in]  in1-gradient tiles (backward)
  float* ring[2];   // TMA stages (forward)
  unsigned long long* bars;
};

__device__ __forceinline__ int al4(int v) { return (v + 3) & ~3; }

__device__ __forceinline__ S3 carve3(const PlanHdr& h, const uint32_t* __restrict__ blob, uint32_t* smem, int stage_floats,
                                     bool backward) {
  for (int i = threadIdx.x; i < h.blob_words; i += blockDim.x) smem[i] = blob[i];
  S3 s;
  s.paths = reinterpret_cast<const PathDev*>(smem + h.off_paths);
  s.cg = reinterpret_cast<const float*>(smem + h.off_cg);
  s.mdesc = reinterpret_cast<const int*>(smem + h.off_mdesc);
  s.vwtasks = reinterpret_cast<const int2*>(smem + h.off_vwtasks);
  float* f = reinterpret_cast<float*>(smem + h.blob_words);
  const int msz = al4(h.te * h.m_size), ysz = al4(h.te * h.d_y);
  s.M[0] = f; s.M[1] = f + msz; f += 2 * msz;
  s.ysh[0] = f; s.ysh[1] = f + ysz; f += 2 * ysz;
  s.wacc = f; f += al4(h.w_numel);
  if (backward) {
    const int gsz = al4(h.te * h.d_in);
    s.gxacc[0] = f; s.gxacc[1] = f + gsz; f += 2 * gsz;
    s.ring[0] = s.ring[1] = nullptr;
  } else {
    s.gxacc[0] = s.gxacc[1] = nullptr;
    s.ring[0] = f; s.ring[1] = f + stage_floats; f += 2 * stage_floats;
  }
  s.bars = reinterpret_cast<unsigned long long*>(f);
  return s;
}

#define EQF3_DISPATCH(val, NAME, ...)                        \
  switch (val) {                                             \
    case 1: { constexpr int NAME = 1; __VA_ARGS__; } break;  \
    case 3: { constexpr int NAME = 3; __VA_ARGS__; } break;  \
    case 5: { constexpr int NAME = 5; __VA_ARGS__; } break;  \
    case 7: { constexpr int NAME = 7; __VA_ARGS__; } break;  \
    default: break;                                          \
  }

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 lds4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, const float4& v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 z4() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void fma4s(float4& acc, const float4& a, float b) {
  acc.x = fmaf(a.x, b, acc.x); acc.y = fmaf(a.y, b, acc.y); acc.z = fmaf(a.z, b, acc.z); acc.w = fmaf(a.w, b, acc.w);
}
__device__ __forceinline__ void fma4v(float4& acc, const float4& a, const float4& b) {
  acc.x = fmaf(a.x, b.x, acc.x); acc.y = fmaf(a.y, b.y, acc.y); acc.z = fmaf(a.z, b.z, acc.z); acc.w = fmaf(a.w, b.w, acc.w);
}

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_init(unsigned long long* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(bar)), "r"(count));
}
__device__ __forceinline__ void bar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void bar_expect(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_1d(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(s32(dst)), "l"(src), "r"(bytes), "r"(s32(bar)) : "memory");
}
__device__ __forceinline__ void bar_wait(unsigned long long* bar, uint32_t parity) {
  for (unsigned it = 0; it < (1u << 28); ++it) {   // bounded: a lost completion traps instead of hanging the box
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(s32(bar)), "r"(parity) : "memory");
    if (ok) return;
  }
  __trap();
}

// fold the harmonics of one tile into M (division-free: edge loop outside, element loop inside)
__device__ __forceinline__ void fold_tile(const PlanHdr& h, const S3& s, const float* ysh, float* M) {
  for (int te = 0; te < h.te; ++te) {
    const float* yy = ysh + te * h.d_y;
    float* Mt = M + te * h.m_size;
    for (int m = threadIdx.x; m < h.m_size; m += blockDim.x) {
      const int desc = s.mdesc[m];
      const PathDev& P = s.paths[desc >> 8];
      const int i = (desc >> 4) & 15, k = desc & 15;
      const float* c = s.cg + P.cg_off + i * P.d2 * P.d3 + k;
      float acc = 0.f;
      for (int j = 0; j < P.d2; ++j) acc = fmaf(c[j * P.d3], yy[P.y_off + j], acc);
      Mt[m] = acc;
    }
  }
}

__device__ __forceinline__ float load_y_elem(const PlanHdr& h, const float* __restrict__ y, long long e0, long long E) {
  const int i = threadIdx.x;
  if (i >= h.te * h.d_y) return 0.f;
  const long long gi = e0 * h.d_y + i;
  return (gi < E * h.d_y) ? __ldg(y + gi) : 0.f;
}

struct Lane3 { int te; int u; bool ok; };
__device__ __forceinline__ Lane3 lane3(const PlanHdr& h, int xb, int2 task, int lane, long long e0, long long E) {
  const int lpe = h.in1_lpe[xb];
  const int sh = h.in1_lpe_shift[xb];
  int sub, v;
  if (sh >= 0) { sub = lane >> sh; v = lane & (lpe - 1); }
  else { sub = lane / lpe; v = lane - sub * lpe; }
  Lane3 m;
  m.te = (task.y >> 16) + sub;
  m.u = (((task.y & 0xffff) << 5) + v) << 2;
  m.ok = sub < h.in1_epw[xb] && m.te < h.te && (e0 + m.te) < E && m.u < h.in1_mul[xb];
  return m;
}

// ---------------------------------------------------------------------------------------------- forward
template <int D1, int D3>
__device__ __forceinline__ void fwd3_task(const PlanHdr& h, const EdgeArgs& a, const PathDev& P, const Lane3& lm,
                                          long long e0, const float* __restrict__ M, const float* wtile,
                                          const float* xtile) {
  if (!lm.ok) return;
  const long long e = e0 + lm.te;
  float4 xi[D1];
  if (xtile != nullptr) {            // in1 rows staged by TMA: [te][d1][mul] per block
    const float* p = xtile + h.te * h.in1_off[P.xb] + (lm.te * D1) * P.mul + lm.u;
#pragma unroll
    for (int i = 0; i < D1; ++i) xi[i] = lds4(p + i * P.mul);
  } else {
    const long long rs = a.src ? a.src[e] : e;
    const float* p = a.x[P.xb] + (rs * D1) * P.mul + lm.u;
#pragma unroll
    for (int i = 0; i < D1; ++i) xi[i] = ld4(p + (long long)i * P.mul);
    if (a.x2[P.xb] != nullptr) {
      const long long rd = a.dst[e];
      const float* q = a.x2[P.xb] + (rd * D1) * P.mul + lm.u;
#pragma unroll
      for (int i = 0; i < D1; ++i) {
        const float4 t = ld4(q + (long long)i * P.mul);
        xi[i].x += t.x; xi[i].y += t.y; xi[i].z += t.z; xi[i].w += t.w;
      }
    }
  }
  float4 wv;
  if (wtile != nullptr) wv = lds4(wtile + lm.te * h.w_numel + P.w_off + lm.u);
  else wv = ld4(a.w + (a.w_shared ? 0 : e * h.w_numel) + P.w_off + lm.u);
  const float* Mp = M + lm.te * h.m_size + P.m_off;
  const int K = h.out_mul[P.og];
  float* o = a.out[P.og] + (e * D3) * K + P.koff + lm.u;
#pragma unroll
  for (int k = 0; k < D3; ++k) {
    float4 acc = z4();
#pragma unroll
    for (int i = 0; i < D1; ++i) fma4s(acc, xi[i], Mp[i * D3 + k]);
    acc.x *= wv.x; acc.y *= wv.y; acc.z *= wv.z; acc.w *= wv.w;
    st4(o + (long long)k * K, acc);
  }
}

// TMA_X: in1 rows are direct (row e) and staged through the ring; otherwise they are read with LDG (gathered or not)
template <bool TMA_W, bool TMA_X>
__global__ void __launch_bounds__(kThreads, 2) dtp_forward_v3_kernel(PlanHdr h, const uint32_t* __restrict__ blob, EdgeArgs a,
                                                                     int stage_floats) {
  extern __shared__ __align__(128) uint32_t smem_raw[];
  const S3 s = carve3(h, blob, smem_raw, stage_floats, false);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n_tiles = (a.E + h.te - 1) / h.te;
  const int x_off = TMA_W ? h.te * h.w_numel : 0;   // ring stage layout: [w tile][x tile]

  auto issue_stage = [&](long long tile, int b) {   // thread 0 only
    const long long e0 = tile * h.te;
    const long long n = (a.E - e0 < h.te) ? (a.E - e0) : h.te;
    uint32_t bytes = 0;
    if (TMA_W) bytes += (uint32_t)n * h.w_numel * 4u;
    if (TMA_X) bytes += (uint32_t)n * h.d_in * 4u;
    bar_expect(&s.bars[b], bytes);
    if (TMA_W) tma_1d(s.ring[b], a.w + e0 * h.w_numel, (uint32_t)n * h.w_numel * 4u, &s.bars[b]);
    if (TMA_X)
      for (int xb = 0; xb < h.n_in1; ++xb) {
        const int row = h.in1_d[xb] * h.in1_mul[xb];
        tma_1d(s.ring[b] + x_off + h.te * h.in1_off[xb], a.x[xb] + e0 * row, (uint32_t)n * row * 4u, &s.bars[b]);
      }
  };

  __syncthreads();  // tables are in shared memory
  const long long tile0 = blockIdx.x;
  if ((TMA_W || TMA_X) && threadIdx.x == 0) {
    bar_init(&s.bars[0], 1);
    bar_init(&s.bars[1], 1);
    bar_fence_init();
    if (tile0 < n_tiles) issue_stage(tile0, 0);
  }
  // prologue: harmonics of the first tile -> M[0]; harmonics of the second tile -> ysh[1]
  if (tile0 < n_tiles) {
    const float y0 = load_y_elem(h, a.y, tile0 * h.te, a.E);
    const long long t1 = tile0 + gridDim.x;
    const float y1 = (t1 < n_tiles) ? load_y_elem(h, a.y, t1 * h.te, a.E) : 0.f;
    if (threadIdx.x < h.te * h.d_y) { s.ysh[0][threadIdx.x] = y0; s.ysh[1][threadIdx.x] = y1; }
    __syncthreads();
    fold_tile(h, s, s.ysh[0], s.M[0]);
  }
  int it = 0;
  for (long long tile = tile0; tile < n_tiles; tile += gridDim.x, ++it) {
    const int b = it & 1, nb = b ^ 1;
    const long long e0 = tile * h.te;
    const long long nt = tile + gridDim.x, nnt = nt + gridDim.x;
    __syncthreads();   // the one barrier of the tile: M[b], ysh[nb] visible; everybody left tile it-1 (M[nb], ring[nb] free)
    if ((TMA_W || TMA_X) && threadIdx.x == 0 && nt < n_tiles) issue_stage(nt, nb);
    const float ynn = (nnt < n_tiles) ? load_y_elem(h, a.y, nnt * h.te, a.E) : 0.f;   // in flight during the work below
    if (nt < n_tiles) fold_tile(h, s, s.ysh[nb], s.M[nb]);                               // fold for the NEXT tile
    const float* wtile = nullptr;
    const float* xtile = nullptr;
    if (TMA_W || TMA_X) {
      bar_wait(&s.bars[b], (uint32_t)((it >> 1) & 1));
      if (TMA_W) wtile = s.ring[b];
      if (TMA_X) xtile = s.ring[b] + x_off;
    }
    const float* M = s.M[b];
    for (int t = warp; t < h.n_vwtasks; t += kWarps) {
      const int2 task = s.vwtasks[t];
      const PathDev& P = s.paths[task.x];
      const Lane3 lm = lane3(h, P.xb, task, lane, e0, a.E);
      EQF3_DISPATCH(P.d1, D1, EQF3_DISPATCH(P.d3, D3, (fwd3_task<D1, D3>(h, a, P, lm, e0, M, wtile, xtile))));
    }
    // ysh[b] (this tile's harmonics) is dead since M[b] was folded one iteration ago: park tile it+2 there
    if (threadIdx.x < h.te * h.d_y) s.ysh[b][threadIdx.x] = ynn;
  }
}

// ---------------------------------------------------------------------------------------------- backward (grad_x [+ grad_w])
template <int D1, int D3, bool WITH_W>
__device__ __forceinline__ void bwd3_task(const PlanHdr& h, const EdgeArgs& a, const PathDev& P, const Lane3& lm,
                                          long long e0, const float* __restrict__ M, float* gxacc, float* wacc) {
  if (!lm.ok) return;
  const long long e = e0 + lm.te;
  const int K = h.out_mul[P.og];
  const float* gp = a.g[P.og] + (e * D3) * K + P.koff + lm.u;
  float4 gk[D3];
#pragma unroll
  for (int k = 0; k < D3; ++k) gk[k] = ld4(gp + (long long)k * K);
  const float4 wv = ld4(a.w + (a.w_shared ? 0 : e * h.w_numel) + P.w_off + lm.u);
  float4 xi[D1];
  if (WITH_W) {
    const long long rs = a.src ? a.src[e] : e;
    const float* p = a.x[P.xb] + (rs * D1) * P.mul + lm.u;
#pragma unroll
    for (int i = 0; i < D1; ++i) xi[i] = ld4(p + (long long)i * P.mul);
    if (a.x2[P.xb] != nullptr) {
      const long long rd = a.dst[e];
      const float* q = a.x2[P.xb] + (rd * D1) * P.mul + lm.u;
#pragma unroll
      for (int i = 0; i < D1; ++i) {
        const float4 t = ld4(q + (long long)i * P.mul);
        xi[i].x += t.x; xi[i].y += t.y; xi[i].z += t.z; xi[i].w += t.w;
      }
    }
  }
  const float* Mp = M + lm.te * h.m_size + P.m_off;
  float* ga = gxacc + h.te * h.in1_off[P.xb] + (lm.te * D1) * P.mul + lm.u;
  float4 gwv = z4();
#pragma unroll
  for (int i = 0; i < D1; ++i) {
    float4 t = z4();
#pragma unroll
    for (int k = 0; k < D3; ++k) fma4s(t, gk[k], Mp[i * D3 + k]);
    if (WITH_W) fma4v(gwv, xi[i], t);
    float* gi = ga + i * P.mul;
    atomicAdd(gi + 0, wv.x * t.x); atomicAdd(gi + 1, wv.y * t.y); atomicAdd(gi + 2, wv.z * t.z); atomicAdd(gi + 3, wv.w * t.w);
  }
  if (WITH_W) {
    if (a.w_shared) {
      float* wa = wacc + P.w_off + lm.u;
      atomicAdd(wa + 0, gwv.x); atomicAdd(wa + 1, gwv.y); atomicAdd(wa + 2, gwv.z); atomicAdd(wa + 3, gwv.w);
    } else {
      st4(a.gw + e * h.w_numel + P.w_off + lm.u, gwv);
    }
  }
}

__device__ __forceinline__ void flush_gx(const PlanHdr& h, const EdgeArgs& a, float* gxacc, long long e0) {
  // write the finished in1-gradient tile (coalesced float4) and clear it for its next use
  const long long n = (a.E - e0 < h.te) ? (a.E - e0) : h.te;
  for (int xb = 0; xb < h.n_in1; ++xb) {
    const int row = h.in1_d[xb] * h.in1_mul[xb];
    float* src = gxacc + h.te * h.in1_off[xb];
    float* dst = a.gx[xb] + e0 * row;
    const int nv = (int)(n * row) >> 2;
    for (int i = threadIdx.x; i < nv; i += blockDim.x) {
      st4(dst + 4 * i, lds4(src + 4 * i));
      st4(src + 4 * i, z4());
    }
  }
}

template <bool WITH_W>
__global__ void __launch_bounds__(kThreads, 2) dtp_backward_v3_kernel(PlanHdr h, const uint32_t* __restrict__ blob, EdgeArgs a) {
  extern __shared__ __align__(128) uint32_t smem_raw[];
  const S3 s = carve3(h, blob, smem_raw, 0, true);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n_tiles = (a.E + h.te - 1) / h.te;
  for (int i = threadIdx.x; i < 2 * al4(h.te * h.d_in); i += blockDim.x) s.gxacc[0][i] = 0.f;
  if (WITH_W && a.w_shared)
    for (int i = threadIdx.x; i < h.w_numel; i += blockDim.x) s.wacc[i] = 0.f;
  __syncthreads();
  const long long tile0 = blockIdx.x;
  if (tile0 < n_tiles) {
    const float y0 = load_y_elem(h, a.y, tile0 * h.te, a.E);
    const long long t1 = tile0 + gridDim.x;
    const float y1 = (t1 < n_tiles) ? load_y_elem(h, a.y, t1 * h.te, a.E) : 0.f;
    if (threadIdx.x < h.te * h.d_y) { s.ysh[0][threadIdx.x] = y0; s.ysh[1][threadIdx.x] = y1; }
    __syncthreads();
    fold_tile(h, s, s.ysh[0], s.M[0]);
  }
  int it = 0;
  long long prev_e0 = -1;
  for (long long tile = tile0; tile < n_tiles; tile += gridDim.x, ++it) {
    const int b = it & 1, nb = b ^ 1;
    const long long e0 = tile * h.te;
    const long long nt = tile + gridDim.x, nnt = nt + gridDim.x;
    __syncthreads();   // tile it-1 finished: its gradient tile gxacc[nb] is complete, M[nb] is free, M[b]/ysh[nb] visible
    const float ynn = (nnt < n_tiles) ? load_y_elem(h, a.y, nnt * h.te, a.E) : 0.f;
    if (prev_e0 >= 0) flush_gx(h, a, s.gxacc[nb], prev_e0);
    if (nt < n_tiles) fold_tile(h, s, s.ysh[nb], s.M[nb]);
    const float* M = s.M[b];
    for (int t = warp; t < h.n_vwtasks; t += kWarps) {
      const int2 task = s.vwtasks[t];
      const PathDev& P = s.paths[task.x];
      const Lane3 lm = lane3(h, P.xb, task, lane, e0, a.E);
      EQF3_DISPATCH(P.d1, D1, EQF3_DISPATCH(P.d3, D3, (bwd3_task<D1, D3, WITH_W>(h, a, P, lm, e0, M, s.gxacc[b], s.wacc))));
    }
    if (threadIdx.x < h.te * h.d_y) s.ysh[b][threadIdx.x] = ynn;
    prev_e0 = e0;
  }
  __syncthreads();
  if (prev_e0 >= 0) flush_gx(h, a, s.gxacc[(it - 1) & 1], prev_e0);
  if (WITH_W && a.w_shared) {
    for (int i = threadIdx.x; i < h.w_numel; i += blockDim.x) a.gw[(long long)blockIdx.x * h.w_numel + i] = s.wacc[i];
  }
}

// ---------------------------------------------------------------------------------------------- host side
template <typename K>
static int smem3(K kernel, size_t bytes) {
  if (bytes <= 48 * 1024) return EQF_OK;
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

static size_t base_words3(const PlanHdr& h) {
  auto a4 = [](size_t v) { return (v + 3) & ~(size_t)3; };
  return (size_t)h.blob_words + 2 * a4((size_t)h.te * h.m_size) + 2 * a4((size_t)h.te * h.d_y) + a4(h.w_numel);
}

int launch_forward_v3(const EqfPlan* plan, const EdgeArgs& a, cudaStream_t stream) {
  const PlanHdr& h = plan->hdr;
  const bool tma_w = !a.w_shared;
  const bool tma_x = (a.src == nullptr && a.x2[0] == nullptr);
  const int stage_floats = (tma_w ? h.te * h.w_numel : 0) + (tma_x ? h.te * h.d_in : 0);
  const size_t smem = 4 * (base_words3(h) + 2 * (size_t)stage_floats) + 32;
  if (smem > 220 * 1024) { set_error("v3 forward: tile does not fit in shared memory"); return EQF_ERR_UNSUPPORTED; }
  const long long n_tiles = (a.E + h.te - 1) / h.te;
  int per_sm = (int)(220 * 1024 / smem);
  per_sm = per_sm < 1 ? 1 : (per_sm > 2 ? 2 : per_sm);
  long long grid = (long long)plan->sm_count * per_sm;
  if (grid > n_tiles) grid = n_tiles;
  int rc;
#define EQF3_LAUNCH_FWD(W, X)                                                                                      \
  do {                                                                                                             \
    if ((rc = smem3(dtp_forward_v3_kernel<W, X>, smem)) != EQF_OK) return rc;                                      \
    dtp_forward_v3_kernel<W, X><<<(unsigned)grid, kThreads, smem, stream>>>(plan->hdr, plan->d_blob, a, stage_floats); \
  } while (0)
  if (tma_w && tma_x) EQF3_LAUNCH_FWD(true, true);
  else if (tma_w) EQF3_LAUNCH_FWD(true, false);
  else if (tma_x) EQF3_LAUNCH_FWD(false, true);
  else EQF3_LAUNCH_FWD(false, false);
#undef EQF3_LAUNCH_FWD
  return check_cuda(cudaGetLastError(), "dtp_forward_v3_kernel launch");
}

int backward_v3_grid(const EqfPlan* plan, long long E) {
  const long long n_tiles = (E + plan->hdr.te - 1) / plan->hdr.te;
  const long long cap = (long long)plan->sm_count * 2;
  return (int)(n_tiles < cap ? (n_tiles > 0 ? n_tiles : 1) : cap);
}

int launch_backward_v3(const EqfPlan* plan, const EdgeArgs& a, bool with_w, cudaStream_t stream) {
  const PlanHdr& h = plan->hdr;
  const size_t smem = 4 * (base_words3(h) + 2 * (((size_t)h.te * h.d_in + 3) & ~(size_t)3)) + 32;
  if (smem > 220 * 1024) { set_error("v3 backward: tile does not fit in shared memory"); return EQF_ERR_UNSUPPORTED; }
  const int grid = backward_v3_grid(plan, a.E);
  int rc;
  if (with_w) {
    if ((rc = smem3(dtp_backward_v3_kernel<true>, smem)) != EQF_OK) return rc;
    dtp_backward_v3_kernel<true><<<grid, kThreads, smem, stream>>>(plan->hdr, plan->d_blob, a);
  } else {
    if ((rc = smem3(dtp_backward_v3_kernel<false>, smem)) != EQF_OK) return rc;
    dtp_backward_v3_kernel<false><<<grid, kThreads, smem, stream>>>(plan->hdr, plan->d_blob, a);
  }
  return check_cuda(cudaGetLastError(), "dtp_backward_v3_kernel launch");
}

}  // namespace eqf
