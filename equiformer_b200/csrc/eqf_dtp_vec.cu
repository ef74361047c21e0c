// eqf_dtp_vec.cu - vectorised (128-bit per lane) DTP kernels with TMA-staged radial weights, sm_90a.
//
// Same math and tables as eqf_dtp.cu; what changes is how bytes move:
//   * every lane owns FOUR consecutive channels: all global accesses are 16-byte LDG/STG, a warp instruction
//     moves 512 contiguous bytes (4 full lines) - 4x fewer memory instructions, 4x more bytes in flight;
//   * a warp covers 32/(mul/4) edges at once when a block has fewer than 128 channels, so no lane idles;
//   * the forward stages the per-edge radial weights - the largest input, W floats per edge, contiguous for a
//     tile of edges - with one `cp.async.bulk` (TMA, UBLKCP in SASS) per tile into a double-buffered shared
//     memory ring, signalled through an mbarrier: the copy of tile t+1 overlaps the math of tile t;
//   * node features are gathered straight from the (L2-resident) node tables with the src/dst indices of the
//     destination-sorted edge list (fuses graph_attention_transformer.py:487 into the operand load).
// Requires every multiplicity to be a multiple of 4 (true for all shipped configs); otherwise the scalar
// kernels of eqf_dtp.cu are used.
#include <mutex>
#include <unordered_map>

#include "eqf_common.cuh"

namespace eqf {

struct VSmem {
  const PathDev* paths;
  const float* cg;
  const int* mdesc;
  const int2* vwtasks;
  const int2* vxtasks;
  const int* xbstart;
  const int* xbpaths;
  float* M;
  float* ysh;
  float* extra;   // [w_numel] accumulators (shared-weight grad) ...
  float* wbuf;    // 2 x [te][w_numel] TMA ring (forward)
  unsigned long long* bars;
};

__device__ __forceinline__ VSmem vcarve(const PlanHdr& h, const uint32_t* __restrict__ blob, uint32_t* smem) {
  for (int i = threadIdx.x; i < h.blob_words; i += blockDim.x) smem[i] = blob[i];
  VSmem s;
  s.paths = reinterpret_cast<const PathDev*>(smem + h.off_paths);
  s.cg = reinterpret_cast<const float*>(smem + h.off_cg);
  s.mdesc = reinterpret_cast<const int*>(smem + h.off_mdesc);
  s.vwtasks = reinterpret_cast<const int2*>(smem + h.off_vwtasks);
  s.vxtasks = reinterpret_cast<const int2*>(smem + h.off_vxtasks);
  s.xbstart = reinterpret_cast<const int*>(smem + h.off_xbstart);
  s.xbpaths = reinterpret_cast<const int*>(smem + h.off_xbpaths);
  float* f = reinterpret_cast<float*>(smem + h.blob_words);
  s.M = f;
  s.ysh = s.M + ((h.te * h.m_size + 3) & ~3);
  s.extra = s.ysh + ((h.te * h.d_y + 3) & ~3);
  s.wbuf = s.extra + ((h.w_numel + 3) & ~3);
  s.bars = reinterpret_cast<unsigned long long*>(s.wbuf + 2 * h.te * h.w_numel);
  return s;
}

__device__ __forceinline__ void vstage_tile(const PlanHdr& h, const VSmem& s, const float* __restrict__ y,
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

#define EQF_VDISPATCH_D(val, NAME, ...)                      \
  switch (val) {                                             \
    case 1: { constexpr int NAME = 1; __VA_ARGS__; } break;  \
    case 3: { constexpr int NAME = 3; __VA_ARGS__; } break;  \
    case 5: { constexpr int NAME = 5; __VA_ARGS__; } break;  \
    case 7: { constexpr int NAME = 7; __VA_ARGS__; } break;  \
    EQF_CASE_D9(NAME, __VA_ARGS__)                           \
    default: break;                                          \
  }

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void stg4(float* p, const float4& v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 f4zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void fma4(float4& acc, const float4& a, float b) {
  acc.x = fmaf(a.x, b, acc.x); acc.y = fmaf(a.y, b, acc.y); acc.z = fmaf(a.z, b, acc.z); acc.w = fmaf(a.w, b, acc.w);
}
__device__ __forceinline__ void fma44(float4& acc, const float4& a, const float4& b) {
  acc.x = fmaf(a.x, b.x, acc.x); acc.y = fmaf(a.y, b.y, acc.y); acc.z = fmaf(a.z, b.z, acc.z); acc.w = fmaf(a.w, b.w, acc.w);
}
__device__ __forceinline__ float4 mul44(const float4& a, const float4& b) {
  return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
}

template <int D1>
__device__ __forceinline__ void load_x4(const EdgeArgs& a, int xb, int mul, long long e, int u, float4 (&xi)[D1]) {
  const long long rs = a.src ? a.src[e] : e;
  const float* p = a.x[xb] + (rs * D1) * mul + u;
#pragma unroll
  for (int i = 0; i < D1; ++i) xi[i] = ldg4(p + (long long)i * mul);
  if (a.x2[xb] != nullptr) {
    const long long rd = a.dst[e];
    const float* q = a.x2[xb] + (rd * D1) * mul + u;
#pragma unroll
    for (int i = 0; i < D1; ++i) {
      const float4 t = ldg4(q + (long long)i * mul);
      xi[i].x += t.x; xi[i].y += t.y; xi[i].z += t.z; xi[i].w += t.w;
    }
  }
}

// lane -> (edge inside the tile, first channel) for a vector task
struct LaneMap { int te; int u; bool ok; };
__device__ __forceinline__ LaneMap lane_map(const PlanHdr& h, int xb, int2 task, int lane, long long e0, long long E) {
  const int lpe = h.in1_lpe[xb], epw = h.in1_epw[xb];
  const int sub = lane / lpe;
  const int v = lane - sub * lpe;
  LaneMap m;
  m.te = (task.y >> 16) + sub;
  m.u = ((task.y & 0xffff) * 32 + v) * 4;
  m.ok = sub < epw && m.te < h.te && (e0 + m.te) < E && m.u < h.in1_mul[xb];
  return m;
}

// ---------------------------------------------------------------------------------------------- TMA helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  // bounded spin: a lost TMA completion traps (launch error) instead of hanging the GPU box
  for (unsigned it = 0; it < (1u << 28); ++it)
    if (mbar_try_wait(bar, parity)) return;
  __trap();
}

// ---------------------------------------------------------------------------------------------- forward
template <int D1, int D3, bool TMA_W>
__device__ __forceinline__ void vfwd_task(const PlanHdr& h, const EdgeArgs& a, const VSmem& s, const PathDev& P,
                                          const LaneMap& lm, long long e0, const float* wtile) {
  if (!lm.ok) return;
  const long long e = e0 + lm.te;
  const MTile<D1, D3> M(s.M + lm.te * h.m_size + P.m_off);
  float4 xi[D1];
  load_x4<D1>(a, P.xb, P.mul, e, lm.u, xi);
  float4 wv;
  if (TMA_W) wv = *reinterpret_cast<const float4*>(wtile + lm.te * h.w_numel + P.w_off + lm.u);
  else wv = ldg4(a.w + (a.w_shared ? 0 : e * h.w_numel) + P.w_off + lm.u);
  const int K = h.out_mul[P.og];
  float* o = a.out[P.og] + (e * D3) * K + P.koff + lm.u;
  if constexpr (MTile<D1, D3>::kInRegs) {
#pragma unroll
    for (int k = 0; k < D3; ++k) {
      float4 acc = f4zero();
#pragma unroll
      for (int i = 0; i < D1; ++i) fma4(acc, xi[i], M(i, k));
      stg4(o + (long long)k * K, mul44(acc, wv));
    }
  } else {
#pragma unroll 1
    for (int k = 0; k < D3; ++k) {
      float4 acc = f4zero();
#pragma unroll
      for (int i = 0; i < D1; ++i) fma4(acc, xi[i], M(i, k));
      stg4(o + (long long)k * K, mul44(acc, wv));
    }
  }
}

template <bool TMA_W>
__global__ void __launch_bounds__(kThreads) dtp_forward_vec_kernel(PlanHdr h, const uint32_t* __restrict__ blob, EdgeArgs a) {
  extern __shared__ __align__(128) uint32_t smem_raw[];
  const VSmem s = vcarve(h, blob, smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n_tiles = (a.E + h.te - 1) / h.te;
  if (TMA_W) {
    if (threadIdx.x == 0) {
      mbar_init(&s.bars[0], 1);
      mbar_init(&s.bars[1], 1);
      fence_mbar_init();
      const long long e0 = (long long)blockIdx.x * h.te;
      if (e0 < a.E) {
        const long long n = (a.E - e0 < h.te) ? (a.E - e0) : h.te;
        const uint32_t bytes = (uint32_t)n * h.w_numel * 4u;
        mbar_expect_tx(&s.bars[0], bytes);
        tma_load_1d(s.wbuf, a.w + e0 * h.w_numel, bytes, &s.bars[0]);
      }
    }
  }
  int it = 0;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
    const long long e0 = tile * h.te;
    __syncthreads();  // every warp finished the previous tile: M/ysh and the other weight buffer are free
    if (TMA_W && threadIdx.x == 0) {
      const long long nt = tile + gridDim.x;
      if (nt < n_tiles) {
        const long long ne0 = nt * h.te;
        const long long n = (a.E - ne0 < h.te) ? (a.E - ne0) : h.te;
        const uint32_t bytes = (uint32_t)n * h.w_numel * 4u;
        const int nb = (it + 1) & 1;
        mbar_expect_tx(&s.bars[nb], bytes);
        tma_load_1d(s.wbuf + (size_t)nb * h.te * h.w_numel, a.w + ne0 * h.w_numel, bytes, &s.bars[nb]);
      }
    }
    vstage_tile(h, s, a.y, e0, a.E);
    const float* wtile = nullptr;
    if (TMA_W) {
      const int b = it & 1;
      mbar_wait(&s.bars[b], (uint32_t)((it >> 1) & 1));
      wtile = s.wbuf + (size_t)b * h.te * h.w_numel;
    }
    for (int t = warp; t < h.n_vwtasks; t += kWarps) {
      const int2 task = s.vwtasks[t];
      const PathDev& P = s.paths[task.x];
      const LaneMap lm = lane_map(h, P.xb, task, lane, e0, a.E);
      EQF_VDISPATCH_D(P.d1, D1, EQF_VDISPATCH_D(P.d3, D3, (vfwd_task<D1, D3, TMA_W>(h, a, s, P, lm, e0, wtile))));
    }
  }
}

// ---------------------------------------------------------------------------------------------- grad_x (+ grad_w)
template <int D1, int D3, bool WITH_W>
__device__ __forceinline__ void vgx_path(const PlanHdr& h, const EdgeArgs& a, const VSmem& s, const PathDev& P,
                                         const LaneMap& lm, long long e, const float4 (&xi)[D1], float4 (&acc)[D1],
                                         float* wacc) {
  const MTile<D1, D3> M(s.M + lm.te * h.m_size + P.m_off);
  const int K = h.out_mul[P.og];
  const float* gp = a.g[P.og] + (e * D3) * K + P.koff + lm.u;
  const float4 wv = ldg4(a.w + (a.w_shared ? 0 : e * h.w_numel) + P.w_off + lm.u);
  float4 gwv = f4zero();
  if constexpr (MTile<D1, D3>::kInRegs) {
    float4 gk[D3];
#pragma unroll
    for (int k = 0; k < D3; ++k) gk[k] = ldg4(gp + (long long)k * K);
#pragma unroll
    for (int i = 0; i < D1; ++i) {
      float4 t = f4zero();
#pragma unroll
      for (int k = 0; k < D3; ++k) fma4(t, gk[k], M(i, k));
      fma44(acc[i], wv, t);
      if (WITH_W) fma44(gwv, xi[i], t);
    }
  } else {                    // one cotangent component at a time (acc[] stays indexed by compile-time i)
#pragma unroll 1
    for (int k = 0; k < D3; ++k) {
      const float4 gk = ldg4(gp + (long long)k * K);
      const float4 wg = mul44(wv, gk);
#pragma unroll
      for (int i = 0; i < D1; ++i) {
        const float c = M(i, k);
        fma4(acc[i], wg, c);
        if (WITH_W) fma44(gwv, xi[i], make_float4(gk.x * c, gk.y * c, gk.z * c, gk.w * c));
      }
    }
  }
  if (WITH_W) {
    if (a.w_shared) {
      float* wa = wacc + P.w_off + lm.u;
      atomicAdd(wa + 0, gwv.x); atomicAdd(wa + 1, gwv.y); atomicAdd(wa + 2, gwv.z); atomicAdd(wa + 3, gwv.w);
    } else {
      stg4(a.gw + e * h.w_numel + P.w_off + lm.u, gwv);
    }
  }
}

template <int D1, bool WITH_W>
__device__ __forceinline__ void vgx_task(const PlanHdr& h, const EdgeArgs& a, const VSmem& s, int xb,
                                         const LaneMap& lm, long long e0, float* wacc) {
  if (!lm.ok) return;
  const long long e = e0 + lm.te;
  const int mul = h.in1_mul[xb];
  float4 xi[D1];
  if (WITH_W) load_x4<D1>(a, xb, mul, e, lm.u, xi);
  float4 acc[D1];
#pragma unroll
  for (int i = 0; i < D1; ++i) acc[i] = f4zero();
  for (int q = s.xbstart[xb]; q < s.xbstart[xb + 1]; ++q) {
    const PathDev& P = s.paths[s.xbpaths[q]];
    EQF_VDISPATCH_D(P.d3, D3, (vgx_path<D1, D3, WITH_W>(h, a, s, P, lm, e, xi, acc, wacc)));
  }
  float* o = a.gx[xb] + (e * D1) * mul + lm.u;
#pragma unroll
  for (int i = 0; i < D1; ++i) stg4(o + (long long)i * mul, acc[i]);
}

template <bool WITH_W>
__global__ void __launch_bounds__(kThreads) dtp_grad_x_vec_kernel(PlanHdr h, const uint32_t* __restrict__ blob, EdgeArgs a) {
  extern __shared__ __align__(128) uint32_t smem_raw[];
  const VSmem s = vcarve(h, blob, smem_raw);
  float* wacc = s.extra;
  if (WITH_W && a.w_shared)
    for (int i = threadIdx.x; i < h.w_numel; i += blockDim.x) wacc[i] = 0.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n_tiles = (a.E + h.te - 1) / h.te;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long e0 = tile * h.te;
    __syncthreads();
    vstage_tile(h, s, a.y, e0, a.E);
    for (int t = warp; t < h.n_vxtasks; t += kWarps) {
      const int2 task = s.vxtasks[t];
      const LaneMap lm = lane_map(h, task.x, task, lane, e0, a.E);
      EQF_VDISPATCH_D(h.in1_d[task.x], D1, (vgx_task<D1, WITH_W>(h, a, s, task.x, lm, e0, wacc)));
    }
  }
  if (WITH_W && a.w_shared) {
    __syncthreads();
    for (int i = threadIdx.x; i < h.w_numel; i += blockDim.x) a.gw[(long long)blockIdx.x * h.w_numel + i] = wacc[i];
  }
}

// ---------------------------------------------------------------------------------------------- host side
// forward: persistent CTAs sized to what fits per SM (each CTA pipelines several tiles through the TMA ring)
static int vgrid_fwd(const EqfPlan* plan, long long E) {
  const long long n_tiles = (E + plan->hdr.te - 1) / plan->hdr.te;
  int per_sm = (int)(220 * 1024 / (plan->smem_bytes_vec_fwd > 0 ? plan->smem_bytes_vec_fwd : 1));
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 8) per_sm = 8;
  const long long cap = (long long)plan->sm_count * per_sm;
  return (int)(n_tiles < cap ? (n_tiles > 0 ? n_tiles : 1) : cap);
}
// backward: same grid as the scalar kernels (rows of the shared-weight partial buffer depend on it)
static int vgrid_bwd(const EqfPlan* plan, long long E) {
  const long long n_tiles = (E + plan->hdr.te - 1) / plan->hdr.te;
  const long long cap = (long long)plan->sm_count * 8;
  return (int)(n_tiles < cap ? (n_tiles > 0 ? n_tiles : 1) : cap);
}

template <typename K>
static int vset_smem(K kernel, size_t bytes) {
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

int launch_forward_vec(const EqfPlan* plan, const EdgeArgs& a, bool tma, cudaStream_t stream) {
  const size_t smem = plan->smem_bytes_vec_fwd;
  int rc;
  if (tma) {
    if ((rc = vset_smem(dtp_forward_vec_kernel<true>, smem)) != EQF_OK) return rc;
    dtp_forward_vec_kernel<true><<<vgrid_fwd(plan, a.E), kThreads, smem, stream>>>(plan->hdr, plan->d_blob, a);
  } else {
    if ((rc = vset_smem(dtp_forward_vec_kernel<false>, smem)) != EQF_OK) return rc;
    dtp_forward_vec_kernel<false><<<vgrid_bwd(plan, a.E), kThreads, plan->smem_bytes_vec_bwd, stream>>>(plan->hdr, plan->d_blob, a);
  }
  return check_cuda(cudaGetLastError(), "dtp_forward_vec_kernel launch");
}

int launch_grad_x_vec(const EqfPlan* plan, const EdgeArgs& a, bool with_w, cudaStream_t stream) {
  const size_t smem = plan->smem_bytes_vec_bwd;
  int rc;
  if (with_w) {
    if ((rc = vset_smem(dtp_grad_x_vec_kernel<true>, smem)) != EQF_OK) return rc;
    dtp_grad_x_vec_kernel<true><<<vgrid_bwd(plan, a.E), kThreads, smem, stream>>>(plan->hdr, plan->d_blob, a);
  } else {
    if ((rc = vset_smem(dtp_grad_x_vec_kernel<false>, smem)) != EQF_OK) return rc;
    dtp_grad_x_vec_kernel<false><<<vgrid_bwd(plan, a.E), kThreads, smem, stream>>>(plan->hdr, plan->d_blob, a);
  }
  return check_cuda(cudaGetLastError(), "dtp_grad_x_vec_kernel launch");
}

}  // namespace eqf
