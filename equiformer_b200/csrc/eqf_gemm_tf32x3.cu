// eqf_gemm_tf32x3.cu - hand-written warpgroup-MMA (wgmma) GEMMs for the per-degree channel-mixing linears (sm_90a).
//
//   forward / data gradient   C[M, N] = A[M, K] * Bt[N, K]^T        M = edges x (2l+1) rows (tall), K, N <= ~1000
//   weight gradient           W[K1, N] = A[R, K1]^T G[R, N]         reduction over the R rows, tiny output
//
// fp32 in HBM, fp32-level accuracy through the 3xTF32 split of eqf_tc.cuh (the weights' hi / lo planes are split once per
// call by a tiny kernel; the A operand is split in registers and fed to wgmma as its register fragment).
//
// Forward: persistent CTAs (one per SM) walking the 128 x BN output tiles, three warpgroups:
//   warpgroup 0      TMA producer (one thread): A tile [128 x 32] and the B hi / lo tiles [BN x 32] of each k-tile
//                    (128-byte rows, SWIZZLE_128B) into a ring of shared-memory stages (full / empty mbarriers); the
//                    ring runs across tile boundaries, so the next tile's operands land while the consumers store
//   warpgroups 1, 2  consumers, 64 rows each: A fragments from shared memory -> hi / lo in registers -> 3 wgmma per
//                    8-deep k-step and 64-column chunk into a k-tile accumulator, added to the running sum in registers.
//                    Two fragment sets: the next k-tile (of this tile or the next) is split while the current one's
//                    MMAs run.  A finished tile goes through a shared-memory staging buffer to TMA stores, which drain
//                    while the consumer computes its next tile.
// Persistence matters for the tall products with a shallow reduction (K = 32, 64: the data gradients of the 1e / 2e
// linears): they are bound by their output stores, and a CTA per tile would wait for a TMA round trip before each store.
// Weight gradient: the same roles over the CTA's slice of the R rows.  Both operands are "MN-major" (the reduction runs
// along the strided dimension), which tf32 wgmma cannot read from shared memory: A^T is read as register fragments
// straight from its swizzled TMA boxes, and the consumers transpose + split each G tile into K-major hi / lo tiles -
// the next stage's while the current stage's MMAs run.
// Every k-tile's MMAs start from a zero accumulator (scale-d 0) and nothing but wgmma writes it between fence and wait,
// so ptxas keeps the MMA chains asynchronous (no injected warpgroup.arrive / wait).
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdlib>
#include <mutex>
#include <string>

#include "eqf_common.cuh"
#include "eqf_tc.cuh"

namespace eqf {
namespace tf32x3 {

using namespace tc;

constexpr int BM = 128;                   // output rows per CTA: two consumer warpgroups of 64
constexpr int BK = kKTile;                // reduction depth per stage (128-byte rows)
constexpr int kRowBytes = BK * 4;
constexpr int kThreads = 384;
constexpr int kConsumerWarps = 8, kConsumerThreads = kConsumerWarps * 32;
constexpr int kSmemBudget = 227 * 1024;
constexpr int kMaxStages = 8;

template <int BN>
struct Smem {
  static constexpr int kABytes = BM * kRowBytes;
  static constexpr int kBBytes = BN * kRowBytes;
  static constexpr int kStageBytes = kABytes + 2 * kBBytes;       // A raw | B hi | B lo
  static constexpr int kOutBytes = 64 * BN * 4;                   // one consumer's C tile: BN / 32 boxes of [64 x 32]
  static constexpr int kStagesRaw = (kSmemBudget - 2048 - 2 * kOutBytes) / kStageBytes;
  static constexpr int kStages = kStagesRaw > kMaxStages ? kMaxStages : kStagesRaw;
  static_assert(kStages >= 2, "tile does not fit shared memory");
  static constexpr int kTotal = kStages * kStageBytes + 2 * kOutBytes + 1024 /* barriers */ + 1024 /* alignment slack */;
};

struct Params {
  long long n_tiles;      // m_blocks * n_blocks, m-block major (the n-blocks of one m-block run side by side: A is
  int n_blocks;           // read from HBM once and from L2 for the other column tiles)
  int N, K;
};

// The consumer's warpgroup tile [64 x BN] into its staging buffer: BN / 32 boxes of [64 rows x 32 columns], 128-byte
// rows, SWIZZLE_128B (the layout the C tensor map stores from).  A warp's float2 writes of one accumulator pair cover
// eight rows x two 16-byte chunks, which the swizzle spreads over all 32 banks: two wavefronts, no conflict.
template <int BN>
__device__ __forceinline__ void stage_acc(const float* acc, uint32_t out, int row_w, int lane) {
#pragma unroll
  for (int i = 0; i < BN / 2; i += 2) {
    const int r = row_w + acc_row(i, lane), c = acc_col(i, lane), cc = c & 31;
    const uint32_t addr = out + (uint32_t)(c >> 5) * 8192u + (uint32_t)r * 128u + (uint32_t)((((cc >> 2) ^ (r & 7)) << 4) + (cc & 3) * 4);
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(acc[i]), "f"(acc[i + 1]) : "memory");
  }
}

// One consumer step: issue the MMAs of the current k-tile (fragments hc / lc), split the next k-tile into hn / ln while
// they run, then retire the stage and promote the k-tile sum; at the last k-tile of a tile, hand the tile to a TMA store.
// Returns false after the consumer's last k-tile.
template <int BN>
struct Consumer {
  using S = Smem<BN>;
  uint8_t* smem;
  uint64_t *full, *empty;
  const CUtensorMap* map_c;
  uint32_t out;                            // this warpgroup's staging buffer
  long long tile, n_tiles;
  int kt, k_tiles, n_blocks, s, row_w, row_wg, lane, wg;
  uint32_t ph;
  bool leader;
  float acc[BN / 2], part[BN / 2];         // running sum, this k-tile's tensor-core sum

  __device__ __forceinline__ bool step(const uint32_t (&hc)[16], const uint32_t (&lc)[16], uint32_t (&hn)[16],
                                       uint32_t (&ln)[16]) {
    const uint32_t st = smem_u32(smem + s * S::kStageBytes);
    mma_ktile_3xtf32<BN, true>(part, hc, lc, st + S::kABytes, st + S::kABytes + S::kBBytes);
    const int s_cur = s;
    const int kt_cur = kt;
    const long long tile_cur = tile;
    if (++s == S::kStages) { s = 0; ph ^= 1; }
    if (++kt == k_tiles) { kt = 0; tile += gridDim.x; }
    const bool more = tile < n_tiles;
    if (more) {
      mbar_wait_hint(&full[s], ph);
      load_a_split(smem_u32(smem + s * S::kStageBytes), row_wg, lane, hn, ln);
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s_cur]);
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = kt_cur == 0 ? part[i] : acc[i] + part[i];
    if (kt_cur == k_tiles - 1) {
      // the staging buffer is free once the previous tile's store has read it
      if (leader) bulk_wait_read();
      named_barrier(wg, 128);
      stage_acc<BN>(acc, out, row_w, lane);
      fence_async_smem();
      named_barrier(wg, 128);
      if (leader) {
        const int m0 = (int)(tile_cur / n_blocks) * BM + (wg - 1) * 64;
        const int n0 = (int)(tile_cur % n_blocks) * BN;
#pragma unroll
        for (int b = 0; b < BN / 32; ++b) tma_store_2d(map_c, n0 + 32 * b, m0, out + (uint32_t)b * 8192u);
        bulk_commit();
      }
    }
    return more;
  }
};

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tf32x3_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_bhi,
                   const __grid_constant__ CUtensorMap map_blo, const __grid_constant__ CUtensorMap map_c, Params p) {
  using S = Smem<BN>;
  constexpr int kStages = S::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* out_base = smem + kStages * S::kStageBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(out_base + 2 * S::kOutBytes);
  uint64_t* empty = full + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int k_tiles = (p.K + BK - 1) / BK;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      prefetch_map(&map_a); prefetch_map(&map_bhi); prefetch_map(&map_blo);
      int s = 0;
      uint32_t ph = 0;
      for (long long tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const int m0 = (int)(tile / p.n_blocks) * BM;
        const int n0 = (int)(tile % p.n_blocks) * BN;
        for (int kt = 0; kt < k_tiles; ++kt) {
          mbar_wait_hint(&empty[s], ph ^ 1);
          uint8_t* st = smem + s * S::kStageBytes;
          mbar_expect_tx(&full[s], (uint32_t)S::kStageBytes);
          tma_load_2d(st, &map_a, kt * BK, m0, &full[s]);
          tma_load_2d(st + S::kABytes, &map_bhi, kt * BK, n0, &full[s]);
          tma_load_2d(st + S::kABytes + S::kBBytes, &map_blo, kt * BK, n0, &full[s]);
          if (++s == kStages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    reg_alloc<232>();
    if ((long long)blockIdx.x >= p.n_tiles) return;
    Consumer<BN> c;
    c.smem = smem; c.full = full; c.empty = empty; c.map_c = &map_c;
    c.out = smem_u32(out_base + (wg - 1) * S::kOutBytes);
    c.tile = blockIdx.x; c.n_tiles = p.n_tiles; c.kt = 0; c.k_tiles = k_tiles; c.n_blocks = p.n_blocks;
    c.s = 0; c.ph = 0; c.lane = lane; c.wg = wg;
    c.row_w = (warp & 3) * 16;
    c.row_wg = (wg - 1) * 64 + c.row_w;                     // first of this warp's 16 rows inside the tile
    c.leader = (threadIdx.x & 127) == 0;
    if (c.leader) prefetch_map(&map_c);
    // two fragment sets: the split of the next k-tile runs while the MMAs of the current one are in flight
    uint32_t h0[16], l0[16], h1[16], l1[16];
    mbar_wait_hint(&full[0], 0);
    load_a_split(smem_u32(smem), c.row_wg, lane, h0, l0);
    while (c.step(h0, l0, h1, l1) && c.step(h1, l1, h0, l0)) {}
    if (c.leader) bulk_wait();
  }
}

// hi / lo planes of the (small) weight operand: hi = w rounded to tf32, lo = w - hi rounded to tf32
__global__ void split_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = w[i];
    const float h = tf32_rn(v);
    hi[i] = h;
    lo[i] = tf32_rn(v - h);
  }
}

// the same split for a weight stored [K, N] (forward product C = A W): the hi / lo planes come out transposed, [N, K]
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

template <int BN>
static int launch(const CUtensorMap& ma, const CUtensorMap& mh, const CUtensorMap& ml, const CUtensorMap& mc, const Params& p,
                  long long m_blocks, int n_blocks, cudaStream_t s) {
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] {
    attr_err = cudaFuncSetAttribute(gemm_tf32x3_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Smem<BN>::kTotal);
  });
  if (attr_err != cudaSuccess) return check_cuda(attr_err, "gemm_tf32x3 smem attribute");
  Params q = p;
  q.n_blocks = n_blocks;
  q.n_tiles = m_blocks * n_blocks;
  const long long sms = device_sms();
  const unsigned grid = (unsigned)(q.n_tiles < sms ? q.n_tiles : sms);
  gemm_tf32x3_kernel<BN><<<grid, kThreads, Smem<BN>::kTotal, s>>>(ma, mh, ml, mc, q);
  return check_cuda(cudaGetLastError(), "gemm_tf32x3_kernel launch");
}

// ================================================================================================ weight gradient
namespace wg {

constexpr int BKR = BK;                   // reduction rows per stage
constexpr int kBoxBytes = BKR * 128;      // one [BKR rows x 32 columns] box of A, SWIZZLE_128B
constexpr int kMaxBN = 128;

struct WParams {
  float* out;
  long long R, rows_per_slice, K1;
  int N;
  int reduce;                             // 1: atomic adds into W[K1, N]; 0: store partial[slice]
};

template <int BN>
struct WSmem {
  static constexpr int kABytes = (BM / 32) * kBoxBytes;           // A: four [BKR x 32] boxes (the CTA's 128 columns of K1)
  static constexpr int kGRawBytes = BKR * BN * 4;                 // G: [BKR x BN] unswizzled rows
  static constexpr int kGBytes = BN * kRowBytes;                  // G^T hi / lo: [BN x BKR] K-major, SWIZZLE_128B
  static constexpr int kStageBytes = kABytes + kGRawBytes + 2 * kGBytes;
  static constexpr int kStagesRaw = (kSmemBudget - 2048) / kStageBytes;
  static constexpr int kStages = kStagesRaw > kMaxStages ? kMaxStages : kStagesRaw;
  static_assert(kStages >= 2, "tile does not fit shared memory");
  static constexpr int kTotal = kStages * kStageBytes + 1024 + 1024;
};

// register fragments of A^T (rows = columns m of A, reduction = rows r of A) from the four swizzled boxes of a stage
__device__ __forceinline__ void load_at_split(uint32_t tile, int row0, int lane, uint32_t (&hi)[16], uint32_t (&lo)[16]) {
  const int g = row0 + (lane >> 2), t = lane & 3;
#pragma unroll
  for (int kb = 0; kb < BKR / 8; ++kb) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int m = g + ((q & 1) ? 8 : 0);
      const int r = kb * 8 + t + ((q & 2) ? 4 : 0);
      const int c = m & 31;
      const uint32_t addr = tile + (uint32_t)(m >> 5) * kBoxBytes + (uint32_t)r * 128u + (uint32_t)((((c >> 2) ^ (r & 7)) << 4) + (c & 3) * 4);
      const float x = lds32(addr);
      const float h = tf32_rn_fast(x);
      hi[kb * 4 + q] = __float_as_uint(h);
      lo[kb * 4 + q] = __float_as_uint(tf32_rn_fast(x - h));
    }
  }
}

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
wgrad_tf32x3_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_g, WParams p) {
  using S = WSmem<BN>;
  constexpr int kStages = S::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * S::kStageBytes);
  uint64_t* empty = full + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wgi = warp >> 2;
  const int m0 = blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const long long r_begin = (long long)blockIdx.z * p.rows_per_slice;
  long long r_end = r_begin + p.rows_per_slice;
  if (r_end > p.R) r_end = p.R;
  const int k_tiles = (int)((r_end - r_begin + BKR - 1) / BKR);    // rows_per_slice % BKR == 0: slices never overlap
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wgi == 0) {
    reg_dealloc<40>();
    if (threadIdx.x == 0) {
      prefetch_map(&map_a); prefetch_map(&map_g);
      for (int kt = 0; kt < k_tiles; ++kt) {
        const int s = kt % kStages;
        mbar_wait_hint(&empty[s], ((kt / kStages) & 1) ^ 1);
        uint8_t* st = smem + s * S::kStageBytes;
        const int r = (int)(r_begin + (long long)kt * BKR);
        mbar_expect_tx(&full[s], (uint32_t)(S::kABytes + S::kGRawBytes));
#pragma unroll
        for (int b = 0; b < BM / 32; ++b) tma_load_2d(st + b * kBoxBytes, &map_a, m0 + 32 * b, r, &full[s]);
        tma_load_2d(st + S::kABytes, &map_g, n0, r, &full[s]);
      }
    }
  } else {
    reg_alloc<232>();
    const int ct = threadIdx.x - 128;                          // 0 .. 255
    const int row_wg = (wgi - 1) * 64 + (warp & 3) * 16;
    // G tile [BKR][BN] of stage s -> G^T hi / lo [BN][BKR]: item (n, 4 reduction rows) = one 16-byte chunk of each plane
    auto transpose_split = [&](int s) {
      const uint32_t g_raw = smem_u32(smem + s * S::kStageBytes) + S::kABytes, g_hi = g_raw + S::kGRawBytes,
                     g_lo = g_hi + S::kGBytes;
      for (int i = ct; i < BN * (BKR / 4); i += kConsumerThreads) {
        const int n = i % BN, rq = i / BN;
        float4 v;
        v.x = lds32(g_raw + (uint32_t)((4 * rq + 0) * BN + n) * 4u);
        v.y = lds32(g_raw + (uint32_t)((4 * rq + 1) * BN + n) * 4u);
        v.z = lds32(g_raw + (uint32_t)((4 * rq + 2) * BN + n) * 4u);
        v.w = lds32(g_raw + (uint32_t)((4 * rq + 3) * BN + n) * 4u);
        float4 h;
        h.x = tf32_rn_fast(v.x); h.y = tf32_rn_fast(v.y); h.z = tf32_rn_fast(v.z); h.w = tf32_rn_fast(v.w);
        const uint32_t off = (uint32_t)n * 128u + (uint32_t)((rq ^ (n & 7)) << 4);
        sts128(g_hi + off, h);
        sts128(g_lo + off, make_float4(tf32_rn_fast(v.x - h.x), tf32_rn_fast(v.y - h.y), tf32_rn_fast(v.z - h.z),
                                       tf32_rn_fast(v.w - h.w)));
      }
      fence_async_smem();
    };
    float acc[BN / 2], part[BN / 2];       // running sum, this k-tile's tensor-core sum
    // One k-tile: its MMAs (fragments hc / lc, G^T planes of its stage) run while the consumers wait for the next stage,
    // transpose + split its G tile and split its A^T fragments into hn / ln; then the k-tile sum is promoted.
    int kt = 0;
    auto step = [&](const uint32_t (&hc)[16], const uint32_t (&lc)[16], uint32_t (&hn)[16], uint32_t (&ln)[16]) {
      const int s = kt % kStages;
      const uint32_t g_hi = smem_u32(smem + s * S::kStageBytes) + S::kABytes + S::kGRawBytes;
      mma_ktile_3xtf32<BN, true>(part, hc, lc, g_hi, g_hi + S::kGBytes);
      const bool more = kt + 1 < k_tiles;
      if (more) {
        const int s1 = (kt + 1) % kStages;
        mbar_wait_hint(&full[s1], ((kt + 1) / kStages) & 1);
        transpose_split(s1);
        load_at_split(smem_u32(smem + s1 * S::kStageBytes), row_wg, lane, hn, ln);
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = kt == 0 ? part[i] : acc[i] + part[i];
      // every consumer's share of the next G^T planes is written before any warpgroup's MMAs read them
      if (more) named_barrier(1, kConsumerThreads);
      ++kt;
      return more;
    };
    uint32_t h0[16], l0[16], h1[16], l1[16];
    mbar_wait_hint(&full[0], 0);
    transpose_split(0);
    load_at_split(smem_u32(smem), row_wg, lane, h0, l0);
    named_barrier(1, kConsumerThreads);
    while (step(h0, l0, h1, l1) && step(h1, l1, h0, l0)) {}
    float* out = p.reduce ? p.out : p.out + (long long)blockIdx.z * p.K1 * p.N;
    store_acc<BN>(acc, out, p.N, m0 + row_wg, p.K1, n0, p.N, lane, p.reduce != 0);
  }
}

struct Shape { int n_tile, n_tiles, m_tiles; long long slices, rows_per_slice; };

static Shape plan(long long R, long long K1, long long N) {
  Shape sh;
  sh.n_tiles = (int)((N + kMaxBN - 1) / kMaxBN);
  sh.n_tile = sh.n_tiles == 1 ? (int)((N + 31) & ~31LL) : kMaxBN;
  sh.m_tiles = (int)((K1 + BM - 1) / BM);
  const long long sms = device_sms();
  long long slices = sms / ((long long)sh.m_tiles * sh.n_tiles);     // one wave of CTAs (one CTA per SM)
  if (slices < 1) slices = 1;
  long long rps = (R + slices - 1) / slices;
  if (rps < 64) rps = 64;
  rps = (rps + BKR - 1) / BKR * BKR;
  sh.rows_per_slice = rps;
  sh.slices = (R + rps - 1) / rps;                                    // every slice non-empty
  return sh;
}

template <int BN>
static int launch(const CUtensorMap& ma, const CUtensorMap& mg, const WParams& p, const Shape& sh, cudaStream_t s) {
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] {
    attr_err = cudaFuncSetAttribute(wgrad_tf32x3_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, WSmem<BN>::kTotal);
  });
  if (attr_err != cudaSuccess) return check_cuda(attr_err, "wgrad_tf32x3 smem attribute");
  dim3 grid((unsigned)sh.m_tiles, (unsigned)sh.n_tiles, (unsigned)sh.slices);
  wgrad_tf32x3_kernel<BN><<<grid, kThreads, WSmem<BN>::kTotal, s>>>(ma, mg, p);
  return check_cuda(cudaGetLastError(), "wgrad_tf32x3_kernel launch");
}

}  // namespace wg
}  // namespace tf32x3
}  // namespace eqf

using namespace eqf;

// C[M, N] = A[M, K] (row-major, lda) x W, 3xTF32 on wgmma.  The weight operand is either Bt[N, K] (b_is_kn = 0, row
// stride ldb >= K: data gradient, W = Bt^T) or B[K, N] (b_is_kn = 1, row stride ldb >= N: forward, W = B).  `split` is
// device scratch of 2 * N * K floats for its hi / lo planes.  Pointers 16-byte aligned, K, lda, ldc multiples of 4.
extern "C" int eqf_gemm_tf32x3(const float* A, const float* Bt, float* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                               int64_t ldb, int64_t ldc, int32_t b_is_kn, float* split, void* stream) {
  using namespace eqf::tf32x3;
  if (M <= 0 || N <= 0) return EQF_OK;
  if (!A || !Bt || !C || !split) { set_error("eqf_gemm_tf32x3: null pointer"); return EQF_ERR_INVALID; }
  if (K <= 0) { set_error("eqf_gemm_tf32x3: K must be positive"); return EQF_ERR_INVALID; }
  if ((((uintptr_t)A | (uintptr_t)C | (uintptr_t)split) & 15) || ((K | lda | ldc) & 3) || lda < K || ldc < N ||
      ldb < (b_is_kn ? N : K)) {
    set_error("eqf_gemm_tf32x3: operands must be 16-byte aligned, K and leading dimensions multiples of 4");
    return EQF_ERR_INVALID;
  }
  if (K > 0x7fffffffLL || N > 0x7fffffffLL) { set_error("eqf_gemm_tf32x3: K / N too large"); return EQF_ERR_UNSUPPORTED; }
  cudaStream_t s = (cudaStream_t)stream;
  float* hi = split;
  float* lo = split + N * K;
  {
    const long long n = N * K;
    const unsigned blocks = (unsigned)((n + 255) / 256 < 1056 ? (n + 255) / 256 : 1056);
    if (b_is_kn) split_transpose_kernel<<<blocks, 256, 0, s>>>(Bt, ldb, hi, lo, N, K);
    else if (ldb == K) split_kernel<<<blocks, 256, 0, s>>>(Bt, hi, lo, n);
    else { set_error("eqf_gemm_tf32x3: Bt must be packed (ldb == K)"); return EQF_ERR_UNSUPPORTED; }
  }
  int rc = check_cuda(cudaGetLastError(), "split_kernel launch");
  if (rc != EQF_OK) return rc;
  // column tiles: as even as possible, at most 128 columns (two register accumulators per thread), rounded up to the
  // instantiated widths
  const long long n_split = (N + 127) / 128;
  const long long per = (N + n_split - 1) / n_split;
  const int bn = per <= 32 ? 32 : per <= 64 ? 64 : per <= 96 ? 96 : 128;
  const int n_blocks = (int)((N + bn - 1) / bn);
  const long long m_blocks = (M + BM - 1) / BM;
  if (M > 0x7fffffffLL) { set_error("eqf_gemm_tf32x3: M too large"); return EQF_ERR_UNSUPPORTED; }
  Params p;
  p.N = (int)N; p.K = (int)K;
  CUtensorMap ma, mh, ml, mc;
  if ((rc = make_map_2d(&ma, A, M, K, lda, BM, BK)) != EQF_OK) return rc;
  if ((rc = make_map_2d(&mh, hi, N, K, K, bn, BK)) != EQF_OK) return rc;
  if ((rc = make_map_2d(&ml, lo, N, K, K, bn, BK)) != EQF_OK) return rc;
  if ((rc = make_map_2d(&mc, C, M, N, ldc, 64, 32)) != EQF_OK) return rc;     // the TMA store clips to [M, N]
  switch (bn) {
    case 32: return launch<32>(ma, mh, ml, mc, p, m_blocks, n_blocks, s);
    case 64: return launch<64>(ma, mh, ml, mc, p, m_blocks, n_blocks, s);
    case 96: return launch<96>(ma, mh, ml, mc, p, m_blocks, n_blocks, s);
    default: return launch<128>(ma, mh, ml, mc, p, m_blocks, n_blocks, s);
  }
}

// number of row slices eqf_gemm_tf32x3_wgrad will use (= leading dimension of its `partial` scratch [slices, K1, N])
extern "C" int64_t eqf_gemm_tf32x3_wgrad_slices(int64_t R, int64_t K1, int64_t N) {
  if (R <= 0 || K1 <= 0 || N <= 0) return 0;
  return eqf::tf32x3::wg::plan(R, K1, N).slices;
}

static int wgrad_impl(const float* A, const float* G, float* out, bool reduce, int64_t R, int64_t K1, int64_t N,
                      int64_t lda, int64_t ldg, void* stream, const char* who) {
  using namespace eqf::tf32x3;
  if (R <= 0 || K1 <= 0 || N <= 0) return EQF_OK;
  if (!A || !G || !out) { set_error(std::string(who) + ": null pointer"); return EQF_ERR_INVALID; }
  if ((((uintptr_t)A | (uintptr_t)G | (uintptr_t)out) & 15) || ((K1 | N | lda | ldg) & 3) || lda < K1 || ldg < N) {
    set_error(std::string(who) + ": operands must be 16-byte aligned, dimensions multiples of 4");
    return EQF_ERR_INVALID;
  }
  if (R > 0x7fffffffLL || K1 > 0x7fffffffLL || N > 0x7fffffffLL) {
    set_error(std::string(who) + ": too many rows");
    return EQF_ERR_UNSUPPORTED;
  }
  const wg::Shape sh = wg::plan(R, K1, N);
  wg::WParams p;
  p.out = out; p.R = R; p.rows_per_slice = sh.rows_per_slice; p.K1 = K1; p.N = (int)N; p.reduce = reduce ? 1 : 0;
  CUtensorMap ma, mg;
  int rc;
  if ((rc = make_map_2d(&ma, A, R, K1, lda, wg::BKR, 32)) != EQF_OK) return rc;
  if ((rc = make_map_2d(&mg, G, R, N, ldg, wg::BKR, sh.n_tile, MapKind::kLinear)) != EQF_OK) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  // W is zeroed and every slice's CTA adds its contribution (the order of the slices' additions is not fixed, so the last
  // bits may differ between runs - like the atomic scatter of the reference)
  if (reduce && (rc = check_cuda(cudaMemsetAsync(out, 0, (size_t)K1 * N * sizeof(float), s), "wgrad memset")) != EQF_OK)
    return rc;
  if (sh.n_tile <= 32) return wg::launch<32>(ma, mg, p, sh, s);
  if (sh.n_tile <= 64) return wg::launch<64>(ma, mg, p, sh, s);
  if (sh.n_tile <= 96) return wg::launch<96>(ma, mg, p, sh, s);
  return wg::launch<128>(ma, mg, p, sh, s);
}

// partial[s] = A[rows of slice s, :K1]^T G[rows of slice s, :N]  for every slice s; the weight gradient is the sum over s
// (deterministic with eqf_colsum).  A [R, K1] (lda), G [R, N] (ldg) row-major fp32, 16-byte aligned, dims multiples of 4.
extern "C" int eqf_gemm_tf32x3_wgrad(const float* A, const float* G, float* partial, int64_t R, int64_t K1, int64_t N,
                                     int64_t lda, int64_t ldg, void* stream) {
  return wgrad_impl(A, G, partial, false, R, K1, N, lda, ldg, stream, "eqf_gemm_tf32x3_wgrad");
}

// W[K1, N] (packed) = A^T G directly: W is zeroed and every slice's CTA adds its contribution with fp32 atomics.
// One launch + one memset instead of partials + column sum.
extern "C" int eqf_gemm_tf32x3_wgrad_accumulate(const float* A, const float* G, float* W, int64_t R, int64_t K1, int64_t N,
                                                int64_t lda, int64_t ldg, void* stream) {
  return wgrad_impl(A, G, W, true, R, K1, N, lda, ldg, stream, "eqf_gemm_tf32x3_wgrad_accumulate");
}
