// eqf_fused.cu - K1: the depth-wise tensor product produced ON CHIP as the A operand of the per-degree channel-mixing
// GEMM that follows it (sm_90a).  Reference path: nets/graph_attention_transformer.py:487-496 -
//   message = src[edge_src] + dst[edge_dst]; f = dtp(message, edge_attr, dtp_rad(edge_scalars)); lin(f) / sep_alpha(f)
// (e3nn 'uvu' tensor product -> [E, 3136] in HBM -> 'uvw' einsum = cuBLAS GEMM).  Here, per output degree l3 (group):
//
//   C[(e, k), c] = sum_u f[e, k, u] W[u, c],     f[e, k, u(p, u')] = w[e, p, u'] * sum_i M_p[e][i, k] * x[e, i, u']
//   M_p[e][i, k] = sum_j CG_p[i, j, k] y[e, j]   (the edge's (2 l1 + 1) x (2 l3 + 1) coupling block, channel independent)
//
// and f never reaches HBM.  One CTA per SM, persistent over 128-row x n_tile output tiles (rows = (edge, component)
// pairs of ONE output degree), warp-specialised:
//   warps 0-3, 8-11  consumers     (two warpgroups, 64 rows each) raw A tile -> registers -> a_hi / a_lo register
//                                  fragments -> 3xTF32 wgmma against the weight tiles; accumulator in registers, stored
//                                  to C at the end of the tile (eqf_tc.cuh)
//   warp  4          TMA producer  weight tiles B_hi / B_lo of the k-tile (K-major planes, 128-byte rows) and, for per-edge
//                                  weights, a box of the [E, W] radial-weight matrix - one "operand slot" per k-tile
//   warps 6-7        table helpers ONE ROW BLOCK AHEAD: the block's src / dst rows and harmonics into shared memory, then the
//                                  coupling blocks M_p[e] from the group's CG blocks (double-buffered, tab_ready / tab_free)
//   warps 12-27      DTP producers two sets of 8 warps alternate k-tiles: gather x = A[src] + B[dst] (float4 per lane, node
//                                  tables L2 resident; issued before the handshake), multiply by the radial weights, contract
//                                  with M_p[e] (128-bit shared loads, dense) and write the 128 x 32 raw A tile (SWIZZLE_128B
//                                  row order, conflict-free for the writers and for the consumers' fragment loads)
// Two independent rings: operand slots (TMA -> consumers' MMAs) and raw A tiles (producers -> consumers' fragment loads).
// Register budget (896 threads x 72 at launch): setmaxnreg gives the TMA / helper warpgroup 56 and each consumer
// warpgroup 80; ptxas allocates the consumer within the 72 of the launch, so it holds a 64 x 64 accumulator and the
// split fragments of half a k-tile at a time.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <mutex>
#include <string>
#include <vector>

#include "eqf_common.cuh"
#include "eqf_tc.cuh"

namespace eqf {
namespace fused {

using namespace tc;

constexpr int BM = 128;                 // rows per tile (two consumer warpgroups of 64)
constexpr int BKT = kKTile;             // channels per k-tile: 128-byte rows
constexpr int kRowBytes = BKT * 4;
constexpr int kProducerWarp = 4;
constexpr int kHelperWarp0 = 6, kHelperWarps = 2, kHelperThreads = kHelperWarps * 32;   // table helpers
constexpr int kConsumerWarps = 8;       // warps 0-3 and 8-11
constexpr int kDtpWarp0 = 12, kDtpWarps = 16, kDtpSets = 2, kDtpSetWarps = kDtpWarps / kDtpSets;
constexpr int kDtpSetThreads = kDtpSetWarps * 32;
constexpr int kThreads = (kDtpWarp0 + kDtpWarps) * 32;            // 896
constexpr int kMaxBN = 64;              // output columns per tile
constexpr int kMaxPaths = 16;
constexpr int kMaxTileEdges = 136;      // 128 / d3 + 2 <= 130
constexpr int kMetaInts = 2 * kMaxTileEdges;   // int32 src / dst rows of the tile's edges
constexpr int kMaxStages = 8;
constexpr int kMaxKTiles = 32;          // K <= 1024 channels per output group

// one CG path feeding the output group of this launch (d3 is common to the group)
struct FPath {
  int d1, d2;        // 2 l1 + 1, 2 l2 + 1
  int xb, mul;       // in1 block and its channel count (row of the block = d1 * mul floats)
  int y_off, w_off;  // offsets into the edge_attr row / the weight row
  int cg_off;        // dense CG block [d1][d2][d3] (path weight folded in) inside `cg`
  int koff;          // first channel of the path inside the group's K
  int m_off;         // offset of this path's [d1][d3] block inside one edge's M row
  unsigned long long nz;   // bit (i * d3 + k): CG_p[i, :, k] has a non-zero entry (M_p[e][i, k] can be non-zero)
};

struct FArgs {
  const float* x[EQF_MAX_BLOCKS];
  const float* x2[EQF_MAX_BLOCKS];
  const long long* src;
  const long long* dst;
  const float* y;
  const float* w;
  const float* w_offset;
  const float* cg;
  float* C;              // [M, N] with row stride ldc
  long long ldc;
  long long E, M;        // edges; GEMM rows = E * d3
  int d_y, W, w_shared, d3, n_paths, m_row, K, N;
  int n_tile, n_blocks;
  long long m_blocks;
  long long* dbg;        // optional clock64 timeline of CTA 0: dbg[role * 2048 + n] (eqf_fused_set_timeline)
  // shared-memory layout (bytes), fixed by the host: n_op operand slots (B hi | B lo | weight box) | n_raw raw A tiles |
  // 2 x (M rows + harmonics + node rows) | descriptors | barriers
  int n_op, n_raw, op_bytes, w_tile_off, w_box_rows, tab_bytes, m_buf_floats, y_buf_floats, cg_floats;
  unsigned char kt_path[kMaxKTiles];   // path of each 32-channel k-tile, in channel order
  FPath paths[kMaxPaths];
};

// timeline of CTA 0: role 0 TMA producer, 1 consumer warp 0 (k-tile start / end), 3 consumer warp 0 (tile stored), 4 DTP
// set 0 (first thread: tables ready, then k-tile start / end), 5 table helper (row block start / end)
__device__ __forceinline__ void stamp(const FArgs& a, int role, int& n) {
  if (a.dbg != nullptr && blockIdx.x == 0 && n < 2048) a.dbg[role * 2048 + n] = clock64();
  ++n;
}


template <int BN>
struct FSmem {
  static constexpr int kABytes = BM * kRowBytes;                    // raw A tile written by the DTP warps
  static constexpr int kBBytes = BN * kRowBytes;
  static constexpr int kBarBytes = 1024;
  static constexpr int kBudget = 227 * 1024 - 1024;
};

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void addv(float4& a, const float4& b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
__device__ __forceinline__ void mulv(float4& a, const float4& b) { a.x *= b.x; a.y *= b.y; a.z *= b.z; a.w *= b.w; }
__device__ __forceinline__ void fs(float4& a, const float4& x, float m) {
  a.x = fmaf(x.x, m, a.x); a.y = fmaf(x.y, m, a.y); a.z = fmaf(x.z, m, a.z); a.w = fmaf(x.w, m, a.w);
}

// ring position + phase parity of a circular buffer of barriers (advanced once per k-tile by every role that uses it)
struct Ring {
  int n, idx;
  uint32_t ph;
  __device__ __forceinline__ Ring(int n_) : n(n_), idx(0), ph(0) {}
  __device__ __forceinline__ void next() { if (++idx == n) { idx = 0; ph ^= 1u; } }
};

// One k-tile (32 channels `ch0 ..` of path p) of the raw A tile: thread t of the set's 256 handles edge t / 8 (+32 ...)
// and the four channels 4 (t % 8) of the chunk.  The coupling block of (edge, path) is read with ceil(D1 D3 / 4) 128-bit
// shared loads from its 16-byte aligned slot and contracted densely, i outermost; DIAG = the l2 = 0 paths, whose block is
// m_i delta_ik.  The first pass's gathers are issued BEFORE the warp waits for its raw slot and the weight box, so
// the L2 round trip overlaps the handshake.  `w_tile`: shared-memory address of the [n_e][32] weight box or 0 (shared w).
struct KtWaits { uint64_t* raw_free; uint32_t raw_ph; uint64_t* op_full; uint32_t op_ph; };

template <int D1, int D3, bool DIAG>
__device__ __forceinline__ void dtp_ktile(const FArgs& a, const FPath& p, int ch0, int t, long long e0, int n_e, long long row0,
                                          const int* __restrict__ src_s, const int* __restrict__ dst_s, uint32_t m_addr,
                                          uint32_t raw_addr, uint32_t w_tile, const KtWaits& wt) {
  constexpr int NM = (D1 * D3 + 3) / 4;
  const int c8 = t & 7;
  const int ch = ch0 + c8 * 4;
  const bool gather = a.src != nullptr;
  const float* xa = a.x[p.xb];
  const float* xb = a.x2[p.xb];
  const long long row_floats = (long long)D1 * p.mul;
  float4 woff = make_float4(0.f, 0.f, 0.f, 0.f);
  if (a.w_offset != nullptr) woff = ld4(a.w_offset + p.w_off + ch);
  bool waited = false;
  int el = t >> 3;
#pragma unroll 1
  do {                                   // at least one trip: every warp has to pass the waits
    const bool active = el < n_e;
    const int els = active ? el : 0;
    const long long e = e0 + els;
    const long long rs = gather ? (long long)src_s[els] : e;
    const float* xp = xa + rs * row_floats + ch;
    float4 x[D1];
#pragma unroll
    for (int i = 0; i < D1; ++i) x[i] = ld4(xp + i * p.mul);
    if (xb != nullptr) {
      const float* xq = xb + (long long)dst_s[els] * row_floats + ch;
      float4 x2[D1];
#pragma unroll
      for (int i = 0; i < D1; ++i) x2[i] = ld4(xq + i * p.mul);
#pragma unroll
      for (int i = 0; i < D1; ++i) addv(x[i], x2[i]);
    }
    if (!waited) {
      waited = true;
      mbar_wait_hint(wt.raw_free, wt.raw_ph);
      if (wt.op_full) mbar_wait_hint(wt.op_full, wt.op_ph);
    }
    if (!active) break;
    float4 wv = w_tile != 0 ? lds128(w_tile + (uint32_t)el * 128u + (uint32_t)c8 * 16u) : ld4(a.w + p.w_off + ch);
    addv(wv, woff);
    float m[NM * 4];
    const uint32_t ma = m_addr + (uint32_t)(el * a.m_row + p.m_off) * 4u;
#pragma unroll
    for (int q = 0; q < NM; ++q) {
      const float4 v = lds128(ma + (uint32_t)q * 16u);
      m[4 * q] = v.x; m[4 * q + 1] = v.y; m[4 * q + 2] = v.z; m[4 * q + 3] = v.w;
    }
    float4 f[D3];
    if constexpr (DIAG) {
#pragma unroll
      for (int k = 0; k < D3; ++k) {
        f[k] = x[k];
        mulv(f[k], wv);
        f[k].x *= m[k * D3 + k]; f[k].y *= m[k * D3 + k]; f[k].z *= m[k * D3 + k]; f[k].w *= m[k * D3 + k];
      }
    } else {
#pragma unroll
      for (int k = 0; k < D3; ++k) f[k] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int i = 0; i < D1; ++i) {
#pragma unroll
        for (int k = 0; k < D3; ++k) fs(f[k], x[i], m[i * D3 + k]);
      }
#pragma unroll
      for (int k = 0; k < D3; ++k) mulv(f[k], wv);
    }
    const int rbase = (int)(e * D3 - row0);
#pragma unroll
    for (int k = 0; k < D3; ++k) {
      const int row = rbase + k;
      if ((unsigned)row < (unsigned)BM) sts128(raw_addr + (uint32_t)row * 128u + (uint32_t)((c8 ^ (row & 7)) << 4), f[k]);
    }
    el += kDtpSetThreads / 8;
  } while (el < n_e);
}

template <int D3>
__device__ __forceinline__ void dtp_ktile_d1(const FArgs& a, const FPath& p, int ch0, int t, long long e0, int n_e, long long row0,
                                             const int* src_s, const int* dst_s, uint32_t m_addr, uint32_t raw_addr,
                                             uint32_t w_tile, const KtWaits& wt) {
  if (p.d2 == 1 && p.d1 == D3) {     // l2 = 0: identity coupling (a multiple of it)
    dtp_ktile<D3, D3, true>(a, p, ch0, t, e0, n_e, row0, src_s, dst_s, m_addr, raw_addr, w_tile, wt);
    return;
  }
  switch (p.d1) {
    case 1: dtp_ktile<1, D3, false>(a, p, ch0, t, e0, n_e, row0, src_s, dst_s, m_addr, raw_addr, w_tile, wt); break;
    case 3: dtp_ktile<3, D3, false>(a, p, ch0, t, e0, n_e, row0, src_s, dst_s, m_addr, raw_addr, w_tile, wt); break;
    case 5: dtp_ktile<5, D3, false>(a, p, ch0, t, e0, n_e, row0, src_s, dst_s, m_addr, raw_addr, w_tile, wt); break;
    default: dtp_ktile<7, D3, false>(a, p, ch0, t, e0, n_e, row0, src_s, dst_s, m_addr, raw_addr, w_tile, wt); break;
  }
}


template <int BN, int D3>
__global__ void __launch_bounds__(kThreads, 1)
dtp_gemm_fwd_kernel(const __grid_constant__ CUtensorMap map_bhi, const __grid_constant__ CUtensorMap map_blo,
                    const __grid_constant__ CUtensorMap map_w, const __grid_constant__ FArgs a) {
  using S = FSmem<BN>;
  const int n_op = a.n_op, n_raw = a.n_raw;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* op_base = smem;                                            // [n_op] x (B hi | B lo | radial-weight box)
  uint8_t* raw_base = smem + (size_t)n_op * a.op_bytes;               // [n_raw] x raw A tile
  uint8_t* tab_base = raw_base + (size_t)n_raw * S::kABytes;          // two table buffers: [m_buf_floats] M rows, harmonics, src / dst rows
  int4* mdesc = reinterpret_cast<int4*>(tab_base + 2 * a.tab_bytes);      // per M-row entry: (cg offset, y offset, d2, -)
  float* cg_s = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(mdesc) + ((a.m_row * 16 + 127) & ~127));   // the group's CG blocks
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(cg_s) + ((a.cg_floats * 4 + 127) & ~127));
  uint64_t* op_full = bars;                        // [8] weight tiles and the radial-weight box landed (TMA)
  uint64_t* op_empty = bars + kMaxStages;          // [8] the MMAs that read the slot's weight tiles finished
  uint64_t* raw_ready = bars + 2 * kMaxStages;     // [8] raw A tile written by the DTP set
  uint64_t* raw_free = bars + 3 * kMaxStages;      // [8] the consumers hold the raw tile in registers
  uint64_t* tab_ready = bars + 4 * kMaxStages;     // [2] tables of a row block built (helper warps)
  uint64_t* tab_free = tab_ready + 2;              // [2] the DTP warps finished the row block

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k_tiles = a.K / BKT;
  constexpr int d3 = D3;        // compile-time output degree: one kernel per degree
  const long long n_tiles_total = a.m_blocks * a.n_blocks;
  const bool w_tma = !a.w_shared;

  if (threadIdx.x == kProducerWarp * 32) {
    prefetch_map(&map_bhi); prefetch_map(&map_blo);
    if (w_tma) prefetch_map(&map_w);
    for (int s = 0; s < kMaxStages; ++s) {
      mbar_init(&op_full[s], 1);
      mbar_init(&op_empty[s], kConsumerWarps);
      mbar_init(&raw_ready[s], kDtpSetWarps);
      mbar_init(&raw_free[s], kConsumerWarps);
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(&tab_ready[b], kHelperWarps);
      mbar_init(&tab_free[b], kDtpWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4 || (warp >= 8 && warp < kDtpWarp0)) {
    // ===================================================================================== consumers (warpgroups 0, 2)
    reg_alloc<80>();
    const int row_wg = (warp < 4 ? 0 : 64) + (warp & 3) * 16;     // first of this warp's 16 rows inside the tile
    const bool stamper = threadIdx.x == 0;
    Ring op(n_op), raw(n_raw);
    int n_stamp = 0;
    for (long long tile = blockIdx.x; tile < n_tiles_total; tile += gridDim.x) {
      const long long mb = tile / a.n_blocks;
      const int nb = (int)(tile % a.n_blocks);
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int kt = 0; kt < k_tiles; ++kt, op.next(), raw.next()) {
        mbar_wait_hint(&op_full[op.idx], op.ph);
        mbar_wait_hint(&raw_ready[raw.idx], raw.ph);
        if (stamper) stamp(a, 1, n_stamp);
        // the k-tile in two halves of two 8-deep k-steps: the accumulator and one half's split fragments fit the
        // 72-register launch budget of the 896-thread CTA, so ptxas keeps the MMAs of a half asynchronous
        const uint32_t raw_tile = smem_u32(raw_base + (size_t)raw.idx * S::kABytes);
        const uint32_t st = smem_u32(op_base + (size_t)op.idx * a.op_bytes);
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          uint32_t hi[8], lo[8];
          load_a_split(raw_tile, row_wg, lane, hi, lo, 2 * half);
          if (half == 1) {         // the raw tile is read: hand the slot back to the DTP warps before the last MMAs
            __syncwarp();
            if (lane == 0) mbar_arrive(&raw_free[raw.idx]);
          }
          mma_ktile_3xtf32<BN>(acc, hi, lo, st, st + S::kBBytes, 2 * half);
          wgmma_wait<0>();
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&op_empty[op.idx]);
        if (stamper) stamp(a, 1, n_stamp);
      }
      store_acc<BN>(acc, a.C, a.ldc, mb * BM + row_wg, a.M, nb * BN, a.N, lane, false);
      if (stamper) stamp(a, 3, n_stamp);
    }
  } else if (warp < 8) {
    // ===================================================================================== warpgroup 1: TMA, table helpers
    reg_dealloc<56>();
    if (warp == kProducerWarp) {
      if (lane == 0) {
        Ring op(n_op);
        int n_stamp = 0;
        const uint32_t tx = (uint32_t)(2 * S::kBBytes) + (w_tma ? (uint32_t)(a.w_box_rows * kRowBytes) : 0u);
        for (long long tile = blockIdx.x; tile < n_tiles_total; tile += gridDim.x) {
          const long long mb = tile / a.n_blocks;
          const int nb = (int)(tile % a.n_blocks);
          const int e0 = (int)((mb * BM) / d3);
          for (int kt = 0; kt < k_tiles; ++kt, op.next()) {
            mbar_wait_hint(&op_empty[op.idx], op.ph ^ 1);
            stamp(a, 0, n_stamp);
            uint8_t* st = op_base + (size_t)op.idx * a.op_bytes;
            mbar_expect_tx(&op_full[op.idx], tx);
            tma_load_2d(st, &map_bhi, kt * BKT, nb * BN, &op_full[op.idx]);
            tma_load_2d(st + S::kBBytes, &map_blo, kt * BKT, nb * BN, &op_full[op.idx]);
            if (w_tma) {
              const FPath& p = a.paths[a.kt_path[kt]];
              tma_load_2d(st + a.w_tile_off, &map_w, p.w_off + (kt * BKT - p.koff), e0, &op_full[op.idx]);
            }
          }
        }
      }
    } else if (warp >= kHelperWarp0) {
      // ------------------------------------------------------------------------------------- table helpers (warps 6, 7)
      // One row block AHEAD of the DTP warps: the block's edges (src / dst rows, harmonics) into shared memory, then the
      // coupling blocks M_p[e] = CG_p . y_e, one thread per entry q of the edge's M row (its CG column in registers)
      // walking the block's edges.
      const int ht = threadIdx.x - kHelperWarp0 * 32;          // 0 .. 63
      const int m_row = a.m_row, d_y = a.d_y;
      {
        int off = 0;
        for (int pi = 0; pi < a.n_paths; ++pi) {
          const FPath& p = a.paths[pi];
          const int n = p.d1 * p.d2 * d3;
          for (int i = ht; i < n; i += kHelperThreads) cg_s[off + i] = __ldg(a.cg + p.cg_off + i);
          off += n;
        }
        for (int q = ht; q < m_row; q += kHelperThreads) {
          int pi = 0, cg0 = 0;
          for (int j = 1; j < a.n_paths; ++j) if (q >= a.paths[j].m_off) pi = j;
          for (int j = 0; j < pi; ++j) cg0 += a.paths[j].d1 * a.paths[j].d2 * d3;
          const FPath& p = a.paths[pi];
          const int r = q - p.m_off;
          const int i = r / d3, k = r - i * d3;
          if (i < p.d1) mdesc[q] = make_int4(cg0 + i * p.d2 * d3 + k, p.y_off, p.d2, 0);
          else mdesc[q] = make_int4(0, 0, 0, 0);           // padding of the path's block to a multiple of 4 floats
        }
        named_barrier(2, kHelperThreads);
      }
      const uint32_t cg_addr = smem_u32(cg_s);
      uint32_t tile_it = 0;
      int n_stamp = 0;
      for (long long tile = blockIdx.x; tile < n_tiles_total; tile += gridDim.x, ++tile_it) {
        const long long mb = tile / a.n_blocks;
        const long long row0 = mb * BM;
        const long long e0 = row0 / d3;
        long long e1 = (row0 + BM - 1) / d3 + 1;
        if (e1 > a.E) e1 = a.E;
        const int n_e = (int)(e1 - e0);
        const int b = tile_it & 1;
        mbar_wait_hint(&tab_free[b], ((tile_it >> 1) & 1) ^ 1);
        if (ht == 0) stamp(a, 5, n_stamp);
        float* mw = reinterpret_cast<float*>(tab_base + b * a.tab_bytes);
        float* ybuf = mw + a.m_buf_floats;
        int* ss = reinterpret_cast<int*>(ybuf + a.y_buf_floats);
        int* ds = ss + kMaxTileEdges;
        if (a.src != nullptr) {
          for (int i = ht; i < n_e; i += kHelperThreads) {
            ss[i] = (int)a.src[e0 + i];
            ds[i] = a.dst != nullptr ? (int)a.dst[e0 + i] : 0;
          }
        }
        for (int i = ht; i < n_e * d_y; i += kHelperThreads) ybuf[i] = __ldg(a.y + e0 * d_y + i);
        named_barrier(2, kHelperThreads);
        const uint32_t y_addr = smem_u32(ybuf);
        for (int q = ht; q < m_row; q += kHelperThreads) {
          const int4 dsc = mdesc[q];
          float cgr[kMaxD];
#pragma unroll
          for (int j = 0; j < kMaxD; ++j) cgr[j] = j < dsc.z ? lds32(cg_addr + (uint32_t)(dsc.x + j * d3) * 4u) : 0.f;
#pragma unroll 4
          for (int el = 0; el < n_e; ++el) {
            const uint32_t ya = y_addr + (uint32_t)(el * d_y + dsc.y) * 4u;
            float m = 0.f;
#pragma unroll
            for (int j = 0; j < kMaxD; ++j)
              if (j < dsc.z) m = fmaf(cgr[j], lds32(ya + (uint32_t)j * 4u), m);
            mw[el * m_row + q] = m;
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&tab_ready[b]);
        if (ht == 0) stamp(a, 5, n_stamp);
      }
    }
  } else {
    // ===================================================================================== DTP producers (warpgroups 3-6)
    const int dt = threadIdx.x - kDtpWarp0 * 32;          // 0 .. 511
    const int set = (warp - kDtpWarp0) / kDtpSetWarps;    // which half of the k-tiles
    const int t = dt - set * kDtpSetThreads;              // 0 .. 255 inside the set
    Ring op(n_op), raw(n_raw);
    uint32_t it = 0, tile_it = 0;
    int n_stamp = 0;
    const bool stamper = (t == 0 && set == 0);            // role 4: first thread of set 0
    for (long long tile = blockIdx.x; tile < n_tiles_total; tile += gridDim.x, ++tile_it) {
      const long long mb = tile / a.n_blocks;
      const long long row0 = mb * BM;
      const long long e0 = row0 / d3;
      long long e1 = (row0 + BM - 1) / d3 + 1;
      if (e1 > a.E) e1 = a.E;
      const int n_e = (int)(e1 - e0);
      const int b = tile_it & 1;
      mbar_wait_hint(&tab_ready[b], (tile_it >> 1) & 1);            // the helper warps built this row block's tables
      if (stamper) stamp(a, 4, n_stamp);
      const float* mw = reinterpret_cast<const float*>(tab_base + b * a.tab_bytes);
      const float* ybuf = mw + a.m_buf_floats;
      const int* src_s = reinterpret_cast<const int*>(ybuf + a.y_buf_floats);
      const int* dst_s = src_s + kMaxTileEdges;
      const uint32_t m_addr = smem_u32(mw);
      for (int kt = 0; kt < k_tiles; ++kt, ++it, op.next(), raw.next()) {
        if ((int)(it & 1) != set) continue;               // the two sets alternate k-tiles
        const FPath& p = a.paths[a.kt_path[kt]];
        const int ch0 = kt * BKT - p.koff;
        const uint32_t raw_addr = smem_u32(raw_base + (size_t)raw.idx * S::kABytes);
        const uint32_t w_tile = w_tma ? smem_u32(op_base + (size_t)op.idx * a.op_bytes) + (uint32_t)a.w_tile_off : 0u;
        KtWaits wt;
        wt.raw_free = &raw_free[raw.idx]; wt.raw_ph = raw.ph ^ 1;
        wt.op_full = w_tma ? &op_full[op.idx] : nullptr; wt.op_ph = op.ph;
        if (stamper) stamp(a, 4, n_stamp);
        dtp_ktile_d1<D3>(a, p, ch0, t, e0, n_e, row0, src_s, dst_s, m_addr, raw_addr, w_tile, wt);
        __syncwarp();
        if (lane == 0) mbar_arrive(&raw_ready[raw.idx]);
        if (stamper) stamp(a, 4, n_stamp);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&tab_free[b]);           // this warp no longer reads the row block's tables
    }
  }
}

// ---------------------------------------------------------------------------------------------- one group to HBM
// The same producer for an output group whose linear is too WIDE to fuse (N > 128 columns: every column tile would
// recompute the product): write f_g[e, k, :K] to HBM (the 0e group of the QM9 model is 224 of the 3136 floats per edge) and
// let the wide wgmma GEMM read it.  One CTA = 32 edges: coupling blocks of its edges in shared memory, then the
// group's k-tiles with the thread layout of dtp_ktile (8 lanes x float4 per edge).
template <int D1, int D3>
__device__ __forceinline__ void group_ktile(const FArgs& a, const FPath& p, int ch0, int el, int c8, long long e,
                                            const float* __restrict__ me, float* __restrict__ out) {
  const int ch = ch0 + c8 * 4;
  float4 wv = ld4(a.w + (a.w_shared ? 0 : e * a.W) + p.w_off + ch);
  if (a.w_offset != nullptr) addv(wv, ld4(a.w_offset + p.w_off + ch));
  const long long row_floats = (long long)D1 * p.mul;
  const long long rs = a.src != nullptr ? a.src[e] : e;
  const float* xp = a.x[p.xb] + rs * row_floats + ch;
  float4 x[D1];
#pragma unroll
  for (int i = 0; i < D1; ++i) x[i] = ld4(xp + i * p.mul);
  if (a.x2[p.xb] != nullptr) {
    const float* xq = a.x2[p.xb] + a.dst[e] * row_floats + ch;
#pragma unroll
    for (int i = 0; i < D1; ++i) addv(x[i], ld4(xq + i * p.mul));
  }
#pragma unroll
  for (int i = 0; i < D1; ++i) mulv(x[i], wv);
#pragma unroll
  for (int k = 0; k < D3; ++k) {
    float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < D1; ++i)
      if ((p.nz >> (i * D3 + k)) & 1ull) fs(f, x[i], me[i * D3 + k]);
    *reinterpret_cast<float4*>(out + (e * D3 + k) * a.K + p.koff + ch) = f;
  }
}

template <int D3>
__global__ void __launch_bounds__(256) dtp_group_forward_kernel(const __grid_constant__ FArgs a, float* __restrict__ out) {
  extern __shared__ float msm[];                       // [32][m_row]
  const int t = threadIdx.x, el = t >> 3, c8 = t & 7;
  const int m_row = a.m_row;
  for (long long eb = (long long)blockIdx.x * 32; eb < a.E; eb += (long long)gridDim.x * 32) {
    const int n_e = (int)((a.E - eb) < 32 ? (a.E - eb) : 32);
    __syncthreads();
    for (int idx = t; idx < n_e * m_row; idx += 256) {
      const int ee = idx / m_row, q = idx - ee * m_row;
      int pi = 0;
      for (int j = 1; j < a.n_paths; ++j) if (q >= a.paths[j].m_off) pi = j;
      const FPath& p = a.paths[pi];
      const int r = q - p.m_off;
      const int i = r / D3, k = r - i * D3;
      const float* cg = a.cg + p.cg_off + i * p.d2 * D3 + k;
      const float* yv = a.y + (eb + ee) * a.d_y + p.y_off;
      float m = 0.f;
      for (int j = 0; j < (i < p.d1 ? p.d2 : 0); ++j) m = fmaf(__ldg(cg + j * D3), __ldg(yv + j), m);   // i >= d1: block padding
      msm[idx] = m;
    }
    __syncthreads();
    if (el < n_e) {
      const long long e = eb + el;
      for (int pi = 0; pi < a.n_paths; ++pi) {
        const FPath& p = a.paths[pi];
        const float* me = msm + el * m_row + p.m_off;
        for (int ch0 = 0; ch0 < p.mul; ch0 += BKT) {
          switch (p.d1) {
            case 1: group_ktile<1, D3>(a, p, ch0, el, c8, e, me, out); break;
            case 3: group_ktile<3, D3>(a, p, ch0, el, c8, e, me, out); break;
            case 5: group_ktile<5, D3>(a, p, ch0, el, c8, e, me, out); break;
            default: group_ktile<7, D3>(a, p, ch0, el, c8, e, me, out); break;
          }
        }
      }
    }
  }
}

// hi / lo planes of a weight stored [K, N] (row stride ldw): the planes come out transposed, [N, K] K-major
__global__ void split_transpose_kernel(const float* __restrict__ w, long long ldw, float* __restrict__ hi,
                                       float* __restrict__ lo, long long N, long long K) {
  const long long n_el = N * K;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_el; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / K, k = i - n * K;
    const float v = w[k * ldw + n];
    const float h = tf32_rn(v);
    hi[i] = h;
    lo[i] = tf32_rn(v - h);
  }
}

template <int BN, int D3>
static int launch_fwd_d3(const CUtensorMap& mh, const CUtensorMap& ml, const CUtensorMap& mw, FArgs& a, cudaStream_t s) {
  using S = FSmem<BN>;
  // shared-memory layout: operand slots (B hi | B lo | radial-weight box) | raw A tiles | 2 table buffers | descriptors |
  // barriers.  The rings are independent: an operand slot is held from its TMA to the MMAs that read the weight tiles,
  // a raw tile only from the DTP warps' stores to the consumers' fragment loads.
  const int n_e_max = BM / a.d3 + 2;
  a.w_box_rows = a.w_shared ? 0 : n_e_max;
  a.w_tile_off = 2 * S::kBBytes;
  a.op_bytes = (a.w_tile_off + a.w_box_rows * kRowBytes + 1023) & ~1023;
  a.m_buf_floats = (n_e_max * a.m_row + 31) & ~31;
  a.y_buf_floats = (n_e_max * a.d_y + 31) & ~31;
  a.cg_floats = 0;
  for (int i = 0; i < a.n_paths; ++i) a.cg_floats += a.paths[i].d1 * a.paths[i].d2 * a.d3;
  a.tab_bytes = ((a.m_buf_floats + a.y_buf_floats) * 4 + kMetaInts * 4 + 127) & ~127;
  const int fixed = 2 * a.tab_bytes + ((a.m_row * 16 + 127) & ~127) + ((a.cg_floats * 4 + 127) & ~127) + S::kBarBytes;
  int n_raw = 0, n_op = 0;
  for (int r = 4; r >= 2 && n_raw == 0; --r) {             // prefer 4 raw tiles (two per DTP set) if >= r operand slots remain
    const int o = (S::kBudget - fixed - r * S::kABytes) / a.op_bytes;
    if (o >= r || (r == 2 && o >= 2)) { n_raw = r; n_op = o; }
  }
  if (n_raw == 0) { set_error("fused DTP: the tile does not fit shared memory"); return EQF_ERR_UNSUPPORTED; }
  if (n_op > kMaxStages) n_op = kMaxStages;
  a.n_raw = n_raw; a.n_op = n_op;
  const int total = n_op * a.op_bytes + n_raw * S::kABytes + fixed + 1024;
  static std::mutex mtx;
  static int attr_bytes = 0;
  {
    std::lock_guard<std::mutex> lock(mtx);
    if (total > attr_bytes) {
      cudaError_t e = cudaFuncSetAttribute(dtp_gemm_fwd_kernel<BN, D3>, cudaFuncAttributeMaxDynamicSharedMemorySize, total);
      if (e != cudaSuccess) return check_cuda(e, "dtp_gemm_fwd smem attribute");
      attr_bytes = total;
    }
  }
  const int sms = device_sms();
  const long long tiles = a.m_blocks * a.n_blocks;
  const int grid = (int)(tiles < sms ? tiles : sms);
  dtp_gemm_fwd_kernel<BN, D3><<<grid, kThreads, total, s>>>(mh, ml, mw, a);
  return check_cuda(cudaGetLastError(), "dtp_gemm_fwd_kernel launch");
}

template <int BN>
static int launch_fwd(const CUtensorMap& mh, const CUtensorMap& ml, const CUtensorMap& mw, FArgs& a, cudaStream_t s) {
  switch (a.d3) {
    case 1: return launch_fwd_d3<BN, 1>(mh, ml, mw, a, s);
    case 3: return launch_fwd_d3<BN, 3>(mh, ml, mw, a, s);
    case 5: return launch_fwd_d3<BN, 5>(mh, ml, mw, a, s);
    default: return launch_fwd_d3<BN, 7>(mh, ml, mw, a, s);
  }
}

// paths of output group `group`, in channel order; returns the number of paths or a negative error
static int collect_paths(const EqfPlan* plan, int group, FArgs& a) {
  const PlanHdr& h = plan->hdr;
  if (group < 0 || group >= h.n_out) { set_error("fused DTP: output group out of range"); return EQF_ERR_INVALID; }
  const PathDev* pd = reinterpret_cast<const PathDev*>(plan->blob.data() + h.off_paths);
  std::vector<const PathDev*> ps;
  for (int p = 0; p < h.n_paths; ++p) if (pd[p].og == group) ps.push_back(&pd[p]);
  for (size_t i = 0; i < ps.size(); ++i)                     // channel order (a handful of paths: insertion sort)
    for (size_t j = i; j > 0 && ps[j]->koff < ps[j - 1]->koff; --j) std::swap(ps[j], ps[j - 1]);
  if (ps.empty() || (int)ps.size() > kMaxPaths) { set_error("fused DTP: unsupported number of paths in the group"); return EQF_ERR_UNSUPPORTED; }
  int koff = 0, m_off = 0;
  for (size_t i = 0; i < ps.size(); ++i) {
    const PathDev& s = *ps[i];
    // the coupling row cgr[kMaxD] spans d2, the non-zero mask nz has 64 bits for d1 x d3, and the group-forward kernel has
    // instances up to d3 = 7: a group with a degree-4 operand or output takes the unfused route (table-walk DTP + GEMM)
    if (s.d1 > kMaxD || s.d2 > kMaxD || s.d3 > kMaxD) {
      set_error("fused DTP: degree-4 paths are not supported (2l+1 <= 7)");
      return EQF_ERR_UNSUPPORTED;
    }
    if (s.koff != koff || s.mul % BKT != 0) {
      set_error("fused DTP: group channels must be covered by paths of multiplicity % 32 == 0");
      return EQF_ERR_UNSUPPORTED;
    }
    FPath& f = a.paths[i];
    f.d1 = s.d1; f.d2 = s.d2; f.xb = s.xb; f.mul = s.mul; f.y_off = s.y_off; f.w_off = s.w_off; f.cg_off = s.cg_off;
    f.koff = s.koff; f.m_off = m_off;
    f.nz = 0;
    const float* cgp = reinterpret_cast<const float*>(plan->blob.data() + h.off_cg) + s.cg_off;
    for (int ii = 0; ii < s.d1; ++ii)
      for (int kk = 0; kk < s.d3; ++kk) {
        bool any = false;
        for (int jj = 0; jj < s.d2; ++jj) any = any || cgp[(ii * s.d2 + jj) * s.d3 + kk] != 0.0f;
        if (any) f.nz |= 1ull << (ii * s.d3 + kk);
      }
    for (int c = 0; c < s.mul / BKT; ++c) {
      if (koff / BKT + c >= kMaxKTiles) { set_error("fused DTP: output group wider than 1024 channels"); return EQF_ERR_UNSUPPORTED; }
      a.kt_path[koff / BKT + c] = (unsigned char)i;
    }
    koff += s.mul;
    m_off += (s.d1 * s.d3 + 3) & ~3;           // every path's [d1][d3] block starts 16-byte aligned (128-bit shared loads)
  }
  a.n_paths = (int)ps.size();
  a.d3 = h.out_d[group];
  a.K = koff;
  a.m_row = m_off;
  if (koff != h.out_mul[group]) { set_error("fused DTP: paths do not cover the output group"); return EQF_ERR_INVALID; }
  if ((BM / a.d3 + 2) * a.m_row * 4 > 40 * 1024) { set_error("fused DTP: coupling blocks of a tile exceed shared memory"); return EQF_ERR_UNSUPPORTED; }
  return a.n_paths;
}

}  // namespace fused
}  // namespace eqf

using namespace eqf;

// 1 when eqf_dtp_linear_fwd can run output group `group` of the plan (multiplicities % 32 == 0, tables fit), else 0
extern "C" int eqf_dtp_linear_supported(const EqfPlan* plan, int32_t group) {
  if (plan == nullptr) return 0;
  fused::FArgs a;
  const PlanHdr& h = plan->hdr;
  for (int b = 0; b < h.n_in1; ++b) if (h.in1_mul[b] % 4 != 0) return 0;
  if (h.w_numel % 4 != 0) return 0;
  return fused::collect_paths(plan, group, a) > 0 ? 1 : 0;
}

static long long* g_fused_dbg = nullptr;
// debugging aid: device buffer of 6 * 2048 int64 that receives CTA 0's clock64 timeline on the next fused launches (NULL = off)
extern "C" void eqf_fused_set_timeline(long long* device_buffer) { g_fused_dbg = device_buffer; }

// operands of one output group -> FArgs (shared by the fused and the group-forward entry points)
static int fill_fargs(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges, int32_t group, eqf::fused::FArgs& a,
                      const char* who) {
  using namespace eqf::fused;
  if (plan == nullptr || op == nullptr) { set_error(std::string(who) + ": null plan / operands"); return EQF_ERR_INVALID; }
  if (!op->y || !op->w) { set_error(std::string(who) + ": null pointer"); return EQF_ERR_INVALID; }
  int rc = ensure_device(plan);
  if (rc != EQF_OK) return rc;
  const PlanHdr& h = plan->hdr;
  rc = collect_paths(plan, group, a);
  if (rc < 0) return rc;
  if ((((uintptr_t)op->w | (uintptr_t)op->w_offset) & 15) || (h.w_numel & 3)) {
    set_error(std::string(who) + ": weights must be 16-byte aligned, weight_numel % 4 == 0");
    return EQF_ERR_INVALID;
  }
  for (int b = 0; b < EQF_MAX_BLOCKS; ++b) { a.x[b] = nullptr; a.x2[b] = nullptr; }
  for (int b = 0; b < h.n_in1; ++b) {
    if (op->x[b] == nullptr || ((uintptr_t)op->x[b] & 15) || ((uintptr_t)op->x2[b] & 15) || (h.in1_mul[b] & 3)) {
      set_error(std::string(who) + ": in1 blocks must be present, 16-byte aligned, multiplicities % 4 == 0");
      return EQF_ERR_INVALID;
    }
    a.x[b] = op->x[b];
    a.x2[b] = op->x2[b];
  }
  a.src = reinterpret_cast<const long long*>(op->src);
  a.dst = reinterpret_cast<const long long*>(op->dst);
  if (a.x2[0] != nullptr && (a.src == nullptr || a.dst == nullptr)) { set_error(std::string(who) + ": x2 needs src and dst"); return EQF_ERR_INVALID; }
  a.y = op->y; a.w = op->w; a.w_offset = op->w_offset; a.w_shared = op->w_shared;
  if (a.w_shared && a.w_offset != nullptr) { set_error(std::string(who) + ": w_offset needs per-edge weights"); return EQF_ERR_INVALID; }
  a.cg = reinterpret_cast<const float*>(plan->d_blob + h.off_cg);
  a.C = nullptr; a.ldc = 0;
  a.E = n_edges; a.M = n_edges * a.d3; a.d_y = h.d_y; a.W = h.w_numel; a.N = 0;
  if (a.M > 0x7fffffffLL) { set_error(std::string(who) + ": too many rows"); return EQF_ERR_UNSUPPORTED; }
  a.n_tile = a.n_blocks = 0; a.m_blocks = 0;
  a.n_op = a.n_raw = a.op_bytes = a.w_tile_off = a.w_box_rows = a.tab_bytes = a.m_buf_floats = a.y_buf_floats = a.cg_floats = 0;
  a.dbg = g_fused_dbg;
  return EQF_OK;
}

// out[e, k, :K] = DTP_group(x, y; w) for ONE output group of the plan, planar [E][2 l3 + 1][K] (the operand of a wide
// linear that is not worth fusing).  Operands as for eqf_dtp_forward.
extern "C" int eqf_dtp_group_forward(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges, int32_t group,
                                     float* out, void* stream) {
  using namespace eqf::fused;
  if (n_edges <= 0) return EQF_OK;
  if (out == nullptr || ((uintptr_t)out & 15)) { set_error("eqf_dtp_group_forward: bad output pointer"); return EQF_ERR_INVALID; }
  FArgs a;
  int rc = fill_fargs(plan, op, n_edges, group, a, "eqf_dtp_group_forward");
  if (rc != EQF_OK) return rc;
  const size_t smem = (size_t)32 * a.m_row * sizeof(float);
  const long long blocks = (n_edges + 31) / 32;
  const int cap = device_sms() * 8;
  const int grid = (int)(blocks < cap ? blocks : cap);
  cudaStream_t s = (cudaStream_t)stream;
  switch (a.d3) {
    case 1: dtp_group_forward_kernel<1><<<grid, 256, smem, s>>>(a, out); break;
    case 3: dtp_group_forward_kernel<3><<<grid, 256, smem, s>>>(a, out); break;
    case 5: dtp_group_forward_kernel<5><<<grid, 256, smem, s>>>(a, out); break;
    default: dtp_group_forward_kernel<7><<<grid, 256, smem, s>>>(a, out); break;
  }
  return check_cuda(cudaGetLastError(), "dtp_group_forward_kernel launch");
}

// C[(e, k), :N] = DTP_group(x, y; w)[(e, k), :K] @ Wt[:K, :N]   for output group `group` of the plan: the depth-wise tensor
// product (nets/graph_attention_transformer.py:491 / :496) feeds the channel-mixing linear (:492, :494, :496) on chip.
// Operands as for eqf_dtp_forward (gather x = x[src] + x2[dst] when op->src is set; w per edge [E, W] (+ w_offset) or
// shared [W]); Wt row-major [K, N] with row stride ldw; C [E * (2 l3 + 1), N] with row stride ldc; `split` = device
// scratch of 2 * N * K floats.  16-byte aligned pointers, N, ldc multiples of 4.
extern "C" int eqf_dtp_linear_fwd(const EqfPlan* plan, const EqfEdgeOperands* op, int64_t n_edges, int32_t group,
                                  const float* Wt, int64_t N, int64_t ldw, float* C, int64_t ldc, float* split,
                                  void* stream) {
  using namespace eqf::fused;
  if (n_edges <= 0 || N <= 0) return EQF_OK;
  if (!Wt || !C || !split) { set_error("eqf_dtp_linear_fwd: null pointer"); return EQF_ERR_INVALID; }
  FArgs a;
  int rc = fill_fargs(plan, op, n_edges, group, a, "eqf_dtp_linear_fwd");
  if (rc != EQF_OK) return rc;
  const PlanHdr& h = plan->hdr;
  if ((((uintptr_t)C | (uintptr_t)split) & 15) || ((N | ldc) & 3) || ldc < N || ldw < N) {
    set_error("eqf_dtp_linear_fwd: operands must be 16-byte aligned, N and ldc multiples of 4");
    return EQF_ERR_INVALID;
  }
  a.N = (int)N;
  cudaStream_t s = (cudaStream_t)stream;
  const long long K = a.K;
  float* hi = split;
  float* lo = split + N * K;
  {
    const long long n = N * K;
    const unsigned blocks = (unsigned)((n + 255) / 256 < 1056 ? (n + 255) / 256 : 1056);
    split_transpose_kernel<<<blocks, 256, 0, s>>>(Wt, ldw, hi, lo, N, K);
  }
  if ((rc = check_cuda(cudaGetLastError(), "split_transpose_kernel launch")) != EQF_OK) return rc;
  // column tiles of at most 64 (the consumers' accumulators live in registers): every tile recomputes the product
  const int n_blocks = (int)((N + kMaxBN - 1) / kMaxBN);
  const int n_tile = (n_blocks == 1 && N <= 32) ? 32 : kMaxBN;
  a.n_tile = n_tile; a.n_blocks = n_blocks; a.m_blocks = (a.M + BM - 1) / BM;
  a.C = C; a.ldc = ldc;
  CUtensorMap mh, ml, mw;
  if ((rc = make_map_2d(&mh, hi, N, K, K, n_tile, BKT)) != EQF_OK) return rc;
  if ((rc = make_map_2d(&ml, lo, N, K, K, n_tile, BKT)) != EQF_OK) return rc;
  mw = mh;    // placeholder when the weights are shared (never dereferenced)
  // per-edge radial weights: [E, W] row-major, a box of (128 / d3 + 2) edges x 32 channels per k-tile, rows back to back
  if (!a.w_shared && (rc = make_map_2d(&mw, a.w, n_edges, h.w_numel, h.w_numel, BM / a.d3 + 2, BKT, MapKind::kLinear)) != EQF_OK)
    return rc;
  if (n_tile == 32) return launch_fwd<32>(mh, ml, mw, a, s);
  return launch_fwd<64>(mh, ml, mw, a, s);
}
