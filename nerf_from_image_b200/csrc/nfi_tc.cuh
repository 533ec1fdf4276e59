// Hopper (sm_90a) tensor-core, mbarrier and TMA-bulk primitives of the tensor-core kernels
// (hand-written PTX, no CUTLASS).
//
// Layer 1 of the decoder (models/generator.py:294-299: Linear(32->64)) runs as
// D[128 points x 64] = A[128 x 32] * W1^T on the tensor cores (wgmma, two M = 64 halves per
// warpgroup) with fp32 accuracy recovered by the hi/lo split ("3xTF32"):
//     a = a_hi + a_lo,  a_hi = a with the low 13 mantissa bits cleared (exactly
//     representable in TF32), a_lo = a - a_hi (exact in fp32);
//     A*W ~= A_lo*W_hi + A_hi*W_lo + A_hi*W_hi       (error ~2^-21 relative)
// Operands live in shared memory in the canonical K-major SWIZZLE_128B layout (a row of 32 fp32 =
// 128 B = one swizzle row; 8 rows = one 1024-B atom); the accumulator lives in the registers of
// the warpgroup that issued the wgmma.  The softplus epilogue works on those registers and hands
// the hidden activations straight back to layer 2 as register A fragments (wgmma's A operand may
// come from registers): a fragment holds, in each k-block of 8, the hidden units 8kb + 2t and
// 8kb + 2t + 1 of lane t = lane % 4, which wgmma reads as K positions t and t + 4.  The B operand
// of every GEMM whose A is such a fragment is stored with its K positions permuted to match
// (kpos_of_hidden below).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "nfi_layout.h"  // sw128_offset, kpos_of_hidden, afrag_slot

namespace nfi {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(0x20000u)  // suspend-time hint (ns): sleep, do not poll
      : "memory");
  return ok != 0;
}
// Waits for the phase with the given parity.  try_wait suspends the thread in
// hardware for a bounded time; a wait that has not succeeded after ~2 s of SM
// clock is a pipeline bug and traps instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (((++spins) & 63u) == 0 && clock64() - t0 > 4000000000LL) __trap();
  }
}
// Same, with a fixed back-off between polls (timing experiments: NFI_WAIT_NS).
template <int NS>
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
  if (NS <= 0) return mbar_wait(bar, parity);
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (true) {
    __nanosleep(NS);
    if (mbar_try_wait(bar, parity)) return;
    if (((++spins) & 63u) == 0 && clock64() - t0 > 4000000000LL) __trap();
  }
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// TMA bulk copy global -> shared, completion on an mbarrier.
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                             uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ------------------------------------------------------------- fences
// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// named barrier over `count` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor (sm_90): bits [0,14) start address >> 4, [16,30) leading byte
// offset >> 4, [32,46) stride byte offset >> 4, [62,64) layout: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B,
// 3 = SWIZZLE_32B.  K-major: rows = M / N, `sbo` = bytes between 8-row groups (the leading offset
// is unused).  MN-major: rows = K, a row holds 64 / 32 / 16 elements of M / N, `lbo` = bytes
// between such atoms along M / N, `sbo` = bytes between 8-row K groups.  A K step inside a
// swizzle atom adds its byte offset >> 4 to the start address.
constexpr uint32_t kSw128 = 1, kSw64 = 2, kSw32 = 3;
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t layout, uint32_t lbo,
                                              uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)layout << 62;
  return d;
}
// K-major, SWIZZLE_128B, 1024 B between 8-row groups: the fp32 [rows x 32] tiles of this project
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  return gmma_desc(smem_addr, kSw128, 16, 1024);
}
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// register fragments must not be touched by the compiler across an in-flight wgmma
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma wrappers: D[64 x N] (+)= A[64 x K] * B[K x N], fp32 accumulators in registers
// (fragment layout of the PTX ISA: warp w of the warpgroup holds rows 16w + lane/4 and
// 16w + lane/4 + 8, columns 8j + 2 (lane % 4) + {0, 1}: d[4j .. 4j+3]).

__device__ __forceinline__ void wgmma_tf32_ss_n64(float (&d)[32], uint64_t a, uint64_t b, int acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(acc)
      : "memory");
}

__device__ __forceinline__ void wgmma_tf32_rs_n16(float (&d)[8], const uint32_t (&a)[4], uint64_t b,
                                                   int acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %13, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc)
      : "memory");
}

__device__ __forceinline__ void wgmma_tf32_rs_n32(float (&d)[16], const uint32_t (&a)[4], uint64_t b,
                                                   int acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc)
      : "memory");
}

__device__ __forceinline__ void wgmma_tf32_rs_n40(float (&d)[20], const uint32_t (&a)[4], uint64_t b,
                                                   int acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %25, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n40k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19}, {%20, %21, %22, %23}, %24, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc)
      : "memory");
}

__device__ __forceinline__ void wgmma_tf32_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t b,
                                                   int acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc)
      : "memory");
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_ss_n8(float (&d)[4], uint64_t a, uint64_t b, int acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %6, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3}, %4, %5, p, 1, 1, %7, %8;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB)
      : "memory");
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_ss_n16(float (&d)[8], uint64_t a, uint64_t b, int acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB)
      : "memory");
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_ss_n32(float (&d)[16], uint64_t a, uint64_t b, int acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB)
      : "memory");
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_ss_n64(float (&d)[32], uint64_t a, uint64_t b, int acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB)
      : "memory");
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_ss_n96(float (&d)[48], uint64_t a, uint64_t b, int acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %50, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, %51, %52;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB)
      : "memory");
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_ss_n128(float (&d)[64], uint64_t a, uint64_t b, int acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB)
      : "memory");
}

// byte offset of (row, 16-byte chunk) inside a [rows x 64 B] SWIZZLE_64B tile (chunk 0..3) and a
// [rows x 32 B] SWIZZLE_32B tile (chunk 0..1): address bits [4,6) / [4,5) XOR bits [7,9) / [7,8)
__device__ __forceinline__ uint32_t sw64_offset(int row, int chunk) {
  return (uint32_t)(row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4));
}
__device__ __forceinline__ uint32_t sw32_offset(int row, int chunk) {
  return (uint32_t)(row * 32 + ((chunk ^ ((row >> 2) & 1)) << 4));
}

__host__ __device__ __forceinline__ float tf32_hi(float x) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
#else
  return x;
#endif
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2_approx(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// two floats -> packed bf16 pair (round-to-nearest-even), `lo` in the low half (lower address)
__device__ __forceinline__ uint32_t bf16x2_rn(float lo, float hi) {
  uint32_t y;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(y) : "f"(hi), "f"(lo));
  return y;
}

// ------------------------------------------------------------- decoder GEMMs of one M = 64 block
// Layer 1, D[64 x 64] = A W1^T in 3xTF32: 12 wgmma (small terms first).  Arguments are descriptor
// bases of the block's A_hi / A_lo rows and of W1 hi / lo; a K step of 8 tf32 = 32 bytes = +2.
__device__ __forceinline__ void layer1_mb(float (&d)[32], uint64_t a_hi, uint64_t a_lo,
                                          uint64_t w_hi, uint64_t w_lo) {
  wgmma_tf32_ss_n64(d, a_lo, w_hi, 0);
#pragma unroll
  for (int ks = 1; ks < 4; ++ks) wgmma_tf32_ss_n64(d, a_lo + 2 * ks, w_hi + 2 * ks, 1);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) wgmma_tf32_ss_n64(d, a_hi + 2 * ks, w_lo + 2 * ks, 1);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) wgmma_tf32_ss_n64(d, a_hi + 2 * ks, w_hi + 2 * ks, 1);
}
// The same 12 products in the same order with A as register fragments (natural K order: k-block
// kb holds channels 8kb + t at a0 / a1 and 8kb + t + 4 at a2 / a3).
__device__ __forceinline__ void layer1_mb_rs(float (&d)[32], const uint32_t (&a_hi)[4][4],
                                             const uint32_t (&a_lo)[4][4], uint64_t w_hi,
                                             uint64_t w_lo) {
  wgmma_tf32_rs_n64(d, a_lo[0], w_hi, 0);
#pragma unroll
  for (int ks = 1; ks < 4; ++ks) wgmma_tf32_rs_n64(d, a_lo[ks], w_hi + 2 * ks, 1);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) wgmma_tf32_rs_n64(d, a_hi[ks], w_lo + 2 * ks, 1);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) wgmma_tf32_rs_n64(d, a_hi[ks], w_hi + 2 * ks, 1);
}
// A fragments of the 64-row block at `row0` of an fp32 [rows x 32] SWIZZLE_128B tile, in the order
// layer1_mb_rs takes them.  The 8 rows a warp reads at once sit in 8 different 16-byte chunks of
// their 128-byte rows, so each of the 16 loads is free of bank conflicts.
__device__ __forceinline__ void load_afrag_sw128(float (&f)[4][4], const unsigned char* tile,
                                                 int row0, int warp, int lane) {
  const int g = lane >> 2, t = lane & 3;
  const int r = row0 + 16 * warp + g;
#pragma unroll
  for (int kb = 0; kb < 4; ++kb) {
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int row = r + 8 * (s & 1), chunk = 2 * kb + (s >> 1);
      f[kb][s] = *reinterpret_cast<const float*>(tile + sw128_offset(row, chunk) + 4 * t);
    }
  }
}
// Layer 2, D[64 x 16] = H W2^T with H as register fragments (hi / lo, 8 k-blocks): 24 wgmma.
// W2 hi / lo: [16 x 64] as two [16 x 32] SWIZZLE_128B K-blocks of 2048 bytes.
__device__ __forceinline__ void layer2_mb(float (&o)[8], const uint32_t (&hhi)[8][4],
                                          const uint32_t (&hlo)[8][4], uint64_t w2_hi,
                                          uint64_t w2_lo) {
#pragma unroll
  for (int ks = 0; ks < 8; ++ks)
    wgmma_tf32_rs_n16(o, hlo[ks], w2_hi + (ks >> 2) * 128 + (ks & 3) * 2, ks != 0);
#pragma unroll
  for (int ks = 0; ks < 8; ++ks)
    wgmma_tf32_rs_n16(o, hhi[ks], w2_lo + (ks >> 2) * 128 + (ks & 3) * 2, 1);
#pragma unroll
  for (int ks = 0; ks < 8; ++ks)
    wgmma_tf32_rs_n16(o, hhi[ks], w2_hi + (ks >> 2) * 128 + (ks & 3) * 2, 1);
}

// The view-conditioned decoder's layer 2, D[64 x 40] = H W2'^T (32 features, the distance, 7 zero
// columns): the 24 products of layer2_mb on [40 x 32] K-blocks (nfi_layout.h).
__device__ __forceinline__ void layer2_vd_mb(float (&o)[20], const uint32_t (&hhi)[8][4],
                                             const uint32_t (&hlo)[8][4], uint64_t w2_hi,
                                             uint64_t w2_lo) {
  constexpr int kb = kVdW2KBlockBytes >> 4;
#pragma unroll
  for (int ks = 0; ks < 8; ++ks)
    wgmma_tf32_rs_n40(o, hlo[ks], w2_hi + (ks >> 2) * kb + (ks & 3) * 2, ks != 0);
#pragma unroll
  for (int ks = 0; ks < 8; ++ks)
    wgmma_tf32_rs_n40(o, hhi[ks], w2_lo + (ks >> 2) * kb + (ks & 3) * 2, 1);
#pragma unroll
  for (int ks = 0; ks < 8; ++ks)
    wgmma_tf32_rs_n40(o, hhi[ks], w2_hi + (ks >> 2) * kb + (ks & 3) * 2, 1);
}
// Its layer 3, D[64 x 16] = Y W3'^T with the 32 activated features as register fragments: 12 wgmma.
__device__ __forceinline__ void layer3_vd_mb(float (&q)[8], const uint32_t (&yhi)[4][4],
                                             const uint32_t (&ylo)[4][4], uint64_t w3_hi,
                                             uint64_t w3_lo) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) wgmma_tf32_rs_n16(q, ylo[ks], w3_hi + 2 * ks, ks != 0);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) wgmma_tf32_rs_n16(q, yhi[ks], w3_lo + 2 * ks, 1);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) wgmma_tf32_rs_n16(q, yhi[ks], w3_hi + 2 * ks, 1);
}

// split v into TF32 hi / remainder and place both at A-fragment register `slot` of k-block kb
template <int KB>
__device__ __forceinline__ void put_split(uint32_t (&hi)[KB][4], uint32_t (&lo)[KB][4], int kb,
                                          int slot, float v) {
  const float h = tf32_hi(v);
  hi[kb][slot] = __float_as_uint(h);
  lo[kb][slot] = __float_as_uint(v - h);
}

// Hidden activations of a layer-1 accumulator block: h = softplus(D1 + b1), returned split as
// TF32 hi / lo A fragments of layer 2.  PRESCALED: D1 and b1 carry log2(e) (the pipelined
// kernels' weight image), softplus(x) = ln2 * (max(x', 0) + lg2(1 + 2^-|x'|)), x' = x log2 e;
// otherwise softplus(x) = max(x, 0) + ln2 * lg2(1 + 2^(-|x| log2 e)).  Two MUFU ops per unit.
template <bool PRESCALED>
__device__ __forceinline__ float softplus_mufu(float x) {
  if (PRESCALED) {
    float l = ex2_approx(-fabsf(x));
    l = lg2_approx(l + 1.f);
    l = l + fmaxf(x, 0.f);
    return l * 0.6931471805599453f;
  }
  const float ax = fabsf(x) * -1.4426950408889634f;
  const float l = lg2_approx(1.f + ex2_approx(ax));
  return fmaf(l, 0.6931471805599453f, fmaxf(x, 0.f));
}
template <bool PRESCALED>
__device__ __forceinline__ void softplus_frag(const float (&d)[32], const float* __restrict__ b1,
                                              int t, uint32_t (&hi)[8][4], uint32_t (&lo)[8][4]) {
#pragma unroll
  for (int kb = 0; kb < 8; ++kb) {
    const float2 bb = *reinterpret_cast<const float2*>(b1 + 8 * kb + 2 * t);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float h = softplus_mufu<PRESCALED>(d[4 * kb + e] + ((e & 1) ? bb.y : bb.x));
      put_split(hi, lo, kb, afrag_slot(e), h);
    }
  }
}

// An accumulator block of 64 rows x 2N columns (N/8 column blocks) -> rows of a row-major
// shared-memory array (`ld` floats per row; the block's row 0 at `rows`)
template <int R>
__device__ __forceinline__ void store_frag_rows(const float (&d)[R], float* rows, int ld, int warp,
                                                int lane) {
  const int g = lane >> 2, t = lane & 3;
  float* r0 = rows + (16 * warp + g) * ld + 2 * t;
#pragma unroll
  for (int j = 0; j < R / 4; ++j) {
    *reinterpret_cast<float2*>(r0 + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(r0 + 8 * ld + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}

}  // namespace tc
}  // namespace nfi
