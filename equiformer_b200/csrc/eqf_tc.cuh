// eqf_tc.cuh - Hopper (sm_90a) building blocks of the tensor-core kernels: mbarrier, TMA, warpgroup MMA (wgmma) with
// the 3xTF32 split, shared by the per-degree GEMMs (eqf_gemm_tf32x3.cu) and the fused edge kernel (eqf_fused.cu).
//
// 3xTF32: a = a_hi + a_lo with a_hi = a rounded to nearest tf32 and a_lo = a - a_hi, itself rounded to nearest tf32 (the
// tensor core would truncate it), likewise for b;
//   a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi     (the dropped a_lo*b_lo term is ~2^-22 relative)
// The tensor core's fp32 accumulation truncates, so the GEMM kernels sum each 32-deep k-tile in a scratch accumulator and
// add it to the running sum with ordinary (round-to-nearest) fp32 adds.
// The A operand of every product is split in registers and handed to wgmma as its register fragment; the B operand (the
// weights' hi / lo planes, split once per call) is a K-major tile of 128-byte rows in shared memory, written by TMA with
// SWIZZLE_128B.  Everything is __forceinline__ device code or a static host helper.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "eqf_common.cuh"

namespace eqf {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!done);
}
// the same wait with a suspend-time hint (ticks): the warp sleeps in hardware until the phase completes or the limit
// expires, instead of returning after the short default limit and being re-issued
__device__ __forceinline__ void mbar_wait_hint(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity), "r"(0x989680u) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void prefetch_map(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// generic-proxy writes to shared memory become visible to the async proxy (wgmma operand reads, TMA)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// round to nearest tf32 (10-bit mantissa), low 13 bits zero: an unbiased split, unlike masking the raw bits (which is
// what the tensor core does to a raw fp32 operand)
__device__ __forceinline__ float tf32_rn(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// the same rounding (nearest, ties away from zero) in two integer instructions (a NaN still reaches the product
// through lo = x - hi = NaN)
__device__ __forceinline__ float tf32_rn_fast(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
}

__device__ __forceinline__ float lds32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const float4& v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// per-warpgroup register re-allocation (all four warps of the group execute it)
template <int N> __device__ __forceinline__ void reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// named barrier among `threads` threads (id 1..15; id 0 is __syncthreads)
__device__ __forceinline__ void named_barrier(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ---------------------------------------------------------------------------------------------- warpgroup MMA
// shared-memory matrix descriptor of a K-major tile of 128-byte rows, SWIZZLE_128B (8-row groups 1024 bytes apart);
// the tile is 1024-byte aligned, a k-step of 8 tf32 inside the swizzle atom advances the start address by 32 bytes
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t addr) {
  return (uint64_t)((addr >> 4) & 0x3FFF) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x 32] (+)= A[64 x 8] (registers, tf32 fragment) x B[8 x 32] (shared memory, K-major SWIZZLE_128B)
__device__ __forceinline__ void wgmma_rs_n32(float* d, const uint32_t* a, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc));
}
// D[64 x 64] (+)= A[64 x 8] (registers, tf32 fragment) x B[8 x 64] (shared memory, K-major SWIZZLE_128B)
__device__ __forceinline__ void wgmma_rs_n64(float* d, const uint32_t* a, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc));
}

constexpr int kKTile = 32;            // reduction depth of one shared-memory stage: 32 tf32 = one 128-byte row

// Register fragments of the warpgroup's 64 rows of a [rows][32] fp32 tile stored with 128-byte rows, SWIZZLE_128B
// (element (r, c) at r * 128 + ((c / 4) ^ (r % 8)) * 16 + (c % 4) * 4 - what TMA writes), split into hi / lo.
// Fragment of k-step kb (8 columns): {(g, t), (g + 8, t), (g, t + 4), (g + 8, t + 4)}, g = 16 warp + lane / 4, t = lane % 4.
// Conflict-free: the eight row groups of a warp hit eight different 16-byte chunks.  N4 / 4 k-steps from k-step kb0 on (a
// whole k-tile by default; kernels short of registers take it in parts).
template <int N4>
__device__ __forceinline__ void load_a_split(uint32_t tile, int row0, int lane, uint32_t (&hi)[N4], uint32_t (&lo)[N4],
                                             int kb0 = 0) {
  static_assert(N4 % 4 == 0 && N4 <= 4 * (kKTile / 8), "whole 8-deep k-steps of one k-tile");
  const int g = row0 + (lane >> 2), t = lane & 3;
#pragma unroll
  for (int kb = 0; kb < N4 / 4; ++kb) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int r = g + ((q & 1) ? 8 : 0);
      const int c = (kb0 + kb) * 8 + t + ((q & 2) ? 4 : 0);
      const float x = lds32(tile + (uint32_t)r * 128u + (uint32_t)((((c >> 2) ^ (r & 7)) << 4) + (c & 3) * 4));
      const float h = tf32_rn_fast(x);
      hi[kb * 4 + q] = __float_as_uint(h);
      lo[kb * 4 + q] = __float_as_uint(tf32_rn_fast(x - h));
    }
  }
}

// acc[64 x BN] += A[64 x 32] B[32 x BN] in 3xTF32: B hi / lo planes are [BN][32] K-major SWIZZLE_128B tiles at b_hi / b_lo.
// hi / lo hold the fragments of N4 / 4 k-steps from k-step kb0 on (load_a_split).  Column chunks of 64 (and one of 32 when
// BN % 64 == 32); chunk j's accumulators are acc[32 j ..].  Issues the MMAs and commits them as one group; the caller
// waits (wgmma_wait) before touching acc, hi, lo or the B tiles again.
template <int BN, int N4>
__device__ __forceinline__ void mma_ktile_3xtf32(float* acc, const uint32_t (&hi)[N4], const uint32_t (&lo)[N4], uint32_t b_hi,
                                                 uint32_t b_lo, int kb0 = 0) {
  static_assert(BN % 32 == 0 && BN >= 32 && BN <= 256, "BN must be a multiple of 32 up to 256");
  wgmma_fence();
#pragma unroll
  for (int kb = 0; kb < N4 / 4; ++kb) {
    const uint64_t adv = (uint64_t)(((kb0 + kb) * 32) >> 4);
#pragma unroll
    for (int j = 0; j < BN / 64; ++j) {
      const uint64_t dh = smem_desc_sw128(b_hi + (uint32_t)j * 8192u) + adv, dl = smem_desc_sw128(b_lo + (uint32_t)j * 8192u) + adv;
      wgmma_rs_n64(acc + 32 * j, &lo[kb * 4], dh);
      wgmma_rs_n64(acc + 32 * j, &hi[kb * 4], dl);
      wgmma_rs_n64(acc + 32 * j, &hi[kb * 4], dh);
    }
    if constexpr (BN % 64 == 32) {
      constexpr int j = BN / 64;
      const uint64_t dh = smem_desc_sw128(b_hi + (uint32_t)j * 8192u) + adv, dl = smem_desc_sw128(b_lo + (uint32_t)j * 8192u) + adv;
      wgmma_rs_n32(acc + 32 * j, &lo[kb * 4], dh);
      wgmma_rs_n32(acc + 32 * j, &hi[kb * 4], dl);
      wgmma_rs_n32(acc + 32 * j, &hi[kb * 4], dh);
    }
  }
  wgmma_commit();
}

// (row, column) of accumulator i of chunk-local fragment layout: rows g, g + 8 (g = 16 warp + lane / 4), columns in pairs
__device__ __forceinline__ int acc_row(int i, int lane) { return (lane >> 2) + ((i >> 1) & 1) * 8; }
__device__ __forceinline__ int acc_col(int i, int lane) { return 8 * ((i & 31) >> 2) + 2 * (lane & 3) + (i & 1) + 64 * (i >> 5); }

// C[row0 + .., col0 + ..] = acc (warpgroup rows row0 .. row0 + 63 of this warp's 16), clipped to [M, N]; atomic adds when `add`
template <int BN>
__device__ __forceinline__ void store_acc(const float* acc, float* C, long long ldc, long long row0, long long M, int col0, int N,
                                          int lane, bool add) {
#pragma unroll
  for (int i = 0; i < BN / 2; i += 2) {
    const long long r = row0 + acc_row(i, lane);
    const int c = col0 + acc_col(i, lane);
    if (r >= M || c >= N) continue;
    float* p = C + r * ldc + c;
    if (add) {
      atomicAdd(p, acc[i]);
      if (c + 1 < N) atomicAdd(p + 1, acc[i + 1]);
    } else if (c + 1 < N) {
      *reinterpret_cast<float2*>(p) = make_float2(acc[i], acc[i + 1]);
    } else {
      *p = acc[i];
    }
  }
}

// ---------------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline EncodeTiled encode_fn() {
  static EncodeTiled fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess) f = nullptr;
    return reinterpret_cast<EncodeTiled>(f);
  }();
  return fn;
}

enum class MapKind { kSwizzled, kLinear };

// 2-D fp32 tensor [rows, cols] with row stride ld (elements), box = [box_rows, box_cols]; zero fill out of bounds.
// kSwizzled: 128-byte box rows, SWIZZLE_128B (wgmma operands and the register-fragment loads); kLinear: unswizzled rows.
static inline int make_map_2d(CUtensorMap* map, const float* base, long long rows, long long cols, long long ld, int box_rows,
                              int box_cols, MapKind kind = MapKind::kSwizzled) {
  EncodeTiled enc = encode_fn();
  if (enc == nullptr) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return EQF_ERR_CUDA; }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapSwizzle sw = kind == MapKind::kLinear ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B;
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (code " + std::to_string((int)r) + ")"); return EQF_ERR_CUDA; }
  return EQF_OK;
}

static inline int device_sms() {
  int sms = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

}  // namespace tc
}  // namespace eqf
