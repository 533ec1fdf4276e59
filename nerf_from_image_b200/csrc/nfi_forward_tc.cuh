// Forward render kernel, tensor-core variant (NFI_MLP_TC_3XTF32).
//
// CTA = 512 threads = 4 independent "tile groups" of 128 threads (one warpgroup each); a group
// owns one 16x8 pixel tile (thread = ray, exactly as in nfi_forward.cuh) and the four groups of
// a CTA cover a 32x16 pixel block of one image.  One CTA per SM: 16 resident warps, ~195 KB of
// shared memory.
//
// Per sample step and group:
//   1. every thread places its point and computes its 3x(offset, fx, fy) taps;
//   2. the group's four warps gather features cooperatively (8 lanes x float4
//      = one 128-byte channel-last texel per tap) and write them, split into
//      TF32 hi/lo parts, straight into the group's A tiles in the wgmma
//      SWIZZLE_128B K-major layout -- features never exist anywhere else;
//   3. the warpgroup issues, per 64-row half of the tile, 12 wgmma (3xTF32, M=64 N=64 K=32)
//      with the accumulator in registers;
//   4. bias + softplus on those registers; the hidden activations go back to the tensor core as
//      register A fragments, split as H_hi / H_lo;
//   5. 24 more wgmma (N=16, K=64) produce the 1+A decoder outputs, which pass through a
//      [128 x 20] shared-memory tile to the thread that owns the ray;
//   6. density / softmax-palette colour / alpha compositing in registers.
// Decoder weights arrive pre-split and pre-swizzled ("weight image", built by
// prep_weight_image) through ONE TMA bulk copy per CTA.
//
// Hierarchical sampling (run.py:259-335): coarse (t, w, sigma, rgb) go to an
// L2-resident scratch slab; the per-ray sort of the S uniforms and the
// inverse-CDF walk use the group's (idle) A-tile memory as S x 128 columns;
// the S sorted fine depths then join the coarse samples in the slab.
#pragma once
#include "nfi_common.cuh"
#include "nfi_forward.cuh"
#include "nfi_tc.cuh"

namespace nfi {

constexpr int kGroups = 4;
constexpr int kTcThreads = kGroups * kThreads;  // 512
constexpr int kW2Pad = 16;

// weight image (bytes)
constexpr int kWiW1Hi = 0;                 // [64 x 32] SW128, 8 KB
constexpr int kWiW1Lo = 8192;
constexpr int kWiW2Hi = 16384;             // [16 x 64] as two [16 x 32] SW128 K-blocks, 4 KB
constexpr int kWiW2Lo = 20480;
constexpr int kWiB1 = 24576;               // 64 floats
constexpr int kWiB2 = kWiB1 + 256;         // 16 floats
constexpr int kWiBytes = kWiB2 + 64;       // 24896
// shared memory map (bytes from the 1024-aligned base)
constexpr int kSmA = 25600;                // 25 * 1024
constexpr int kSmAGroup = 32768;           // A_hi (16 KB) + A_lo (16 KB); later H_hi k-blocks 0/1
constexpr int kOutLd = 20;                 // decoder-output tile: [128 rays][20] floats per group
constexpr int kSmOut = kSmA + kGroups * kSmAGroup;
constexpr int kSmPal = kSmOut + kGroups * kThreads * kOutLd * 4;
constexpr int kSmBars = kSmPal + 48 * 4;   // 1 mbarrier (weights)
constexpr int kSmTcBytes = kSmBars + 8;

// scratch per group-tile: float4 srgb[S][128], float t[S][128], w[S][128], zf[S][128]
__host__ __device__ inline size_t tc_scratch_floats_per_group(int S) {
  return (size_t)S * kThreads * 7;
}

// Builds the weight image: W1 split into TF32 hi/lo and laid out as the wgmma
// B operand ([64 rows = hidden unit][32 k] fp32, K-major, SWIZZLE_128B), W2
// padded to 16 rows with its K positions in register-fragment order (tc::kpos_of_hidden), biases.
static __global__ void prep_weight_image(const float* __restrict__ w1, const float* __restrict__ b1,
                                  const float* __restrict__ w2, const float* __restrict__ b2,
                                  int nout, unsigned char* __restrict__ img, float scale1,
                                  float pad_b2, float scale2) {
  // scale1: factor folded into layer 1 (W1 and b1); pad_b2: value of the padded
  // layer-2 biases; scale2: factor folded into the colour rows (>= 1) of layer 2.  The
  // pipelined kernel wants log2(e), -1e30, log2(e) (nfi_forward_pipe.cuh); others 1, 0, 1.
  for (int i = threadIdx.x; i < kHid * kC; i += blockDim.x) {
    const int j = i / kC, k = i % kC;  // W1[j][k]
    const float w = w1[i] * scale1;
    const float hi = tc::tf32_hi(w);
    const uint32_t off = tc::sw128_offset(j, k >> 2) + (k & 3) * 4;
    *reinterpret_cast<float*>(img + kWiW1Hi + off) = hi;
    *reinterpret_cast<float*>(img + kWiW1Lo + off) = w - hi;
  }
  for (int i = threadIdx.x; i < kW2Pad * kHid; i += blockDim.x) {
    const int o = i / kHid, j = i % kHid;  // W2[o][j], rows >= nout are zero
    const float w = (o < nout) ? w2[o * kHid + j] * (o >= 1 ? scale2 : 1.f) : 0.f;
    const float hi = tc::tf32_hi(w);
    const int jp = tc::kpos_of_hidden(j);
    const uint32_t off = (jp >> 5) * 2048 + tc::sw128_offset(o, (jp & 31) >> 2) + (jp & 3) * 4;
    *reinterpret_cast<float*>(img + kWiW2Hi + off) = hi;
    *reinterpret_cast<float*>(img + kWiW2Lo + off) = w - hi;
  }
  float* b1i = reinterpret_cast<float*>(img + kWiB1);
  float* b2i = reinterpret_cast<float*>(img + kWiB2);
  for (int i = threadIdx.x; i < kHid; i += blockDim.x) b1i[i] = b1[i] * scale1;
  for (int i = threadIdx.x; i < kW2Pad; i += blockDim.x)
    b2i[i] = (i < nout) ? b2[i] * (i >= 1 ? scale2 : 1.f) : pad_b2;
}

struct PackedTaps {
  uint32_t o[3];  // texel offset of the nw tap | dx << 30 | dy << 31
  float fx[3], fy[3];
};

__device__ __forceinline__ void pack_taps(float gx, float gy, int R, uint32_t& o, float& fx,
                                          float& fy) {
  const float m = (float)(R - 1);
  float ix = (gx + 1.f) * 0.5f * m;
  float iy = (gy + 1.f) * 0.5f * m;
  ix = fminf(m, fmaxf(ix, 0.f));
  iy = fminf(m, fmaxf(iy, 0.f));
  const float x0 = floorf(ix), y0 = floorf(iy);
  fx = ix - x0;
  fy = iy - y0;
  const int xi = (int)x0, yi = (int)y0;
  o = (uint32_t)(yi * R + xi) | ((xi + 1 < R) ? (1u << 30) : 0u) | ((yi + 1 < R) ? (1u << 31) : 0u);
}

__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// interpolates one plane's 4 taps for this lane's 4 channels, accumulating into acc
__device__ __forceinline__ void plane_taps_acc(const float4* __restrict__ plane, uint32_t o,
                                               float fx, float fy, int R, float4& acc,
                                               bool first) {
  const uint32_t o00 = o & 0x3FFFFFFFu;
  const uint32_t dx = (o >> 30) & 1u, dy = (o >> 31) ? (uint32_t)R : 0u;
  const float gx0 = 1.f - fx, gy0 = 1.f - fy;
  const float w00 = gx0 * gy0, w01 = fx * gy0, w10 = gx0 * fy, w11 = fx * fy;
  const float4 a = ldg4(plane + (size_t)o00 * (kC / 4));
  const float4 b = ldg4(plane + (size_t)(o00 + dx) * (kC / 4));
  const float4 c = ldg4(plane + (size_t)(o00 + dy) * (kC / 4));
  const float4 d = ldg4(plane + (size_t)(o00 + dy + dx) * (kC / 4));
  float2 lo = first ? make_float2(0.f, 0.f) : make_float2(acc.x, acc.y);
  float2 hi = first ? make_float2(0.f, 0.f) : make_float2(acc.z, acc.w);
  lo = ffma2(make_float2(a.x, a.y), make_float2(w00, w00), lo);
  hi = ffma2(make_float2(a.z, a.w), make_float2(w00, w00), hi);
  lo = ffma2(make_float2(b.x, b.y), make_float2(w01, w01), lo);
  hi = ffma2(make_float2(b.z, b.w), make_float2(w01, w01), hi);
  lo = ffma2(make_float2(c.x, c.y), make_float2(w10, w10), lo);
  hi = ffma2(make_float2(c.z, c.w), make_float2(w10, w10), hi);
  lo = ffma2(make_float2(d.x, d.y), make_float2(w11, w11), lo);
  hi = ffma2(make_float2(d.z, d.w), make_float2(w11, w11), hi);
  acc = make_float4(lo.x, lo.y, hi.x, hi.y);
}

// Cooperative gather of this warp's 32 points into rows [row0, row0+32) of the
// group's A_hi / A_lo tiles (byte pointers, SWIZZLE_128B layout).
__device__ __forceinline__ void gather_to_tiles(const float* __restrict__ planes_b, int R,
                                                const PackedTaps& tp, unsigned char* a_hi,
                                                unsigned char* a_lo, int row0, int lane) {
  const int q = lane >> 3, k = lane & 7;
  const size_t plane_stride4 = (size_t)R * R * (kC / 4);
  const float4* base = reinterpret_cast<const float4*>(planes_b) + k;
#pragma unroll 2
  for (int g = 0; g < 8; ++g) {
    const int src = 4 * g + q;
    float4 acc;
#pragma unroll
    for (int pl = 0; pl < 3; ++pl) {
      const uint32_t o = __shfl_sync(kFull, tp.o[pl], src);
      const float fx = __shfl_sync(kFull, tp.fx[pl], src);
      const float fy = __shfl_sync(kFull, tp.fy[pl], src);
      plane_taps_acc(base + pl * plane_stride4, o, fx, fy, R, acc, pl == 0);
    }
    const float third = 0.33333334f;  // mean of the three planes (generator.py:328)
    const float4 f = make_float4(acc.x * third, acc.y * third, acc.z * third, acc.w * third);
    const float4 fh = make_float4(tc::tf32_hi(f.x), tc::tf32_hi(f.y), tc::tf32_hi(f.z),
                                  tc::tf32_hi(f.w));
    const float4 fl = make_float4(f.x - fh.x, f.y - fh.y, f.z - fh.z, f.w - fh.w);
    const uint32_t off = tc::sw128_offset(row0 + src, k);
    *reinterpret_cast<float4*>(a_hi + off) = fh;
    *reinterpret_cast<float4*>(a_lo + off) = fl;
  }
}

// Software-pipelined variant of gather_to_tiles: the texel lines of point
// group g+2 are PREFETCHED into L1 (no registers held) while group g is loaded
// (now an L1 hit) and interpolated, so a warp never sits on an L2 round trip.
struct GroupTaps {
  uint32_t off[12];  // float4 index of each tap for this lane (plane and channel quad included)
  float fx[3], fy[3];
};

__device__ __forceinline__ void group_taps(const PackedTaps& tp, int src, int R,
                                           uint32_t plane_stride4, int k, GroupTaps& t) {
#pragma unroll
  for (int pl = 0; pl < 3; ++pl) {
    const uint32_t o = __shfl_sync(kFull, tp.o[pl], src);
    t.fx[pl] = __shfl_sync(kFull, tp.fx[pl], src);
    t.fy[pl] = __shfl_sync(kFull, tp.fy[pl], src);
    const uint32_t o00 = o & 0x3FFFFFFFu;
    const uint32_t dx = (o >> 30) & 1u, dy = (o >> 31) ? (uint32_t)R : 0u;
    const uint32_t b = pl * plane_stride4 + k;
    t.off[4 * pl + 0] = o00 * (kC / 4) + b;
    t.off[4 * pl + 1] = (o00 + dx) * (kC / 4) + b;
    t.off[4 * pl + 2] = (o00 + dy) * (kC / 4) + b;
    t.off[4 * pl + 3] = (o00 + dy + dx) * (kC / 4) + b;
  }
}

__device__ __forceinline__ void group_prefetch(const float4* __restrict__ planes4,
                                               const GroupTaps& t) {
#pragma unroll
  for (int i = 0; i < 12; ++i) tc::prefetch_l1(planes4 + t.off[i]);
}

__device__ __forceinline__ void group_consume(const float4* __restrict__ planes4,
                                              const GroupTaps& t, unsigned char* a_hi,
                                              unsigned char* a_lo, int row, int k) {
  float4 v[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) v[i] = ldg4(planes4 + t.off[i]);
  float2 lo = make_float2(0.f, 0.f), hi = make_float2(0.f, 0.f);
#pragma unroll
  for (int pl = 0; pl < 3; ++pl) {
    const float gx0 = 1.f - t.fx[pl], gy0 = 1.f - t.fy[pl];
    const float w[4] = {gx0 * gy0, t.fx[pl] * gy0, gx0 * t.fy[pl], t.fx[pl] * t.fy[pl]};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4 x = v[4 * pl + j];
      lo = ffma2(make_float2(x.x, x.y), make_float2(w[j], w[j]), lo);
      hi = ffma2(make_float2(x.z, x.w), make_float2(w[j], w[j]), hi);
    }
  }
  const float third = 0.33333334f;
  const float4 f = make_float4(lo.x * third, lo.y * third, hi.x * third, hi.y * third);
  const float4 fh = make_float4(tc::tf32_hi(f.x), tc::tf32_hi(f.y), tc::tf32_hi(f.z),
                                tc::tf32_hi(f.w));
  const float4 fl = make_float4(f.x - fh.x, f.y - fh.y, f.z - fh.z, f.w - fh.w);
  const uint32_t off = tc::sw128_offset(row, k);
  *reinterpret_cast<float4*>(a_hi + off) = fh;
  *reinterpret_cast<float4*>(a_lo + off) = fl;
}

__device__ __forceinline__ void gather_to_tiles_pf(const float* __restrict__ planes_b, int R,
                                                   const PackedTaps& tp, unsigned char* a_hi,
                                                   unsigned char* a_lo, int row0, int lane) {
  const int q = lane >> 3, k = lane & 7;
  const uint32_t plane_stride4 = (uint32_t)R * R * (kC / 4);
  const float4* planes4 = reinterpret_cast<const float4*>(planes_b);
  GroupTaps ta, tb;
  group_taps(tp, q, R, plane_stride4, k, ta);
  group_prefetch(planes4, ta);
  group_taps(tp, 4 + q, R, plane_stride4, k, tb);
  group_prefetch(planes4, tb);
#pragma unroll 1
  for (int g = 0; g < 8; g += 2) {
    group_consume(planes4, ta, a_hi, a_lo, row0 + 4 * g + q, k);
    if (g + 2 < 8) {
      group_taps(tp, 4 * (g + 2) + q, R, plane_stride4, k, ta);
      group_prefetch(planes4, ta);
    }
    group_consume(planes4, tb, a_hi, a_lo, row0 + 4 * (g + 1) + q, k);
    if (g + 3 < 8) {
      group_taps(tp, 4 * (g + 3) + q, R, plane_stride4, k, tb);
      group_prefetch(planes4, tb);
    }
  }
}

__device__ __forceinline__ float4 ldg_nc_volatile(const float4* p) {
  float4 r;  // volatile: the 12 loads of a point group must issue back-to-back, before any use
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

// Gather for the producer warps: per point group (4 points x 8 lanes) the 9 tap
// parameters are shuffled in, the 12 texel loads are ISSUED TOGETHER, then
// interpolated.  (A structure that interleaves loads and FFMA2s leaves only ~4
// loads in flight per warp and serialises ~24 L2 round trips per step.)
__device__ __forceinline__ void gather_to_tiles_deep(const float* __restrict__ planes_b, int R,
                                                     const PackedTaps& tp, unsigned char* a_hi,
                                                     unsigned char* a_lo, int row0, int lane) {
  const int q = lane >> 3, k = lane & 7;
  const uint32_t plane_stride4 = (uint32_t)R * R * (kC / 4);
  const float4* base = reinterpret_cast<const float4*>(planes_b) + k;
#pragma unroll 1
  for (int g = 0; g < 8; ++g) {
    const int src = 4 * g + q;
    uint32_t off[12];
    float fx[3], fy[3];
#pragma unroll
    for (int pl = 0; pl < 3; ++pl) {
      const uint32_t o = __shfl_sync(kFull, tp.o[pl], src);
      fx[pl] = __shfl_sync(kFull, tp.fx[pl], src);
      fy[pl] = __shfl_sync(kFull, tp.fy[pl], src);
      const uint32_t o00 = (o & 0x3FFFFFFFu) * (kC / 4) + pl * plane_stride4;
      const uint32_t dx = ((o >> 30) & 1u) * (kC / 4), dy = (o >> 31) ? (uint32_t)R * (kC / 4) : 0u;
      off[4 * pl + 0] = o00;
      off[4 * pl + 1] = o00 + dx;
      off[4 * pl + 2] = o00 + dy;
      off[4 * pl + 3] = o00 + dy + dx;
    }
    float4 v[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) v[i] = ldg_nc_volatile(base + off[i]);
    float2 lo = make_float2(0.f, 0.f), hi = make_float2(0.f, 0.f);
#pragma unroll
    for (int pl = 0; pl < 3; ++pl) {
      const float gx0 = 1.f - fx[pl], gy0 = 1.f - fy[pl];
      const float w[4] = {gx0 * gy0, fx[pl] * gy0, gx0 * fy[pl], fx[pl] * fy[pl]};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 x = v[4 * pl + j];
        lo = ffma2(make_float2(x.x, x.y), make_float2(w[j], w[j]), lo);
        hi = ffma2(make_float2(x.z, x.w), make_float2(w[j], w[j]), hi);
      }
    }
    const float third = 0.33333334f;
    const float4 f = make_float4(lo.x * third, lo.y * third, hi.x * third, hi.y * third);
    const float4 fh = make_float4(tc::tf32_hi(f.x), tc::tf32_hi(f.y), tc::tf32_hi(f.z),
                                  tc::tf32_hi(f.w));
    const float4 fl = make_float4(f.x - fh.x, f.y - fh.y, f.z - fh.z, f.w - fh.w);
    const uint32_t offs = tc::sw128_offset(row0 + src, k);
    *reinterpret_cast<float4*>(a_hi + offs) = fh;
    *reinterpret_cast<float4*>(a_lo + offs) = fl;
  }
}

// ---------------------------------------------------------------------------
// Lean gather (nfi_forward_pipe.cuh): same arithmetic as gather_to_tiles_deep,
// about half the instructions.  The owner lane of a point pre-multiplies its
// three nw-texel offsets into offsets from the image's plane base in 16-byte units
// (plane index and the 8 units of a texel included; the two border flags ride in
// bits 0/1 of the multiple-of-8 value), so the serving lanes only mask, add and
// widen (one IMAD.WIDE.U32 per address: x16 + base).
// ---------------------------------------------------------------------------
struct ByteTaps {
  uint32_t o[3];  // offset of the nw texel in 16-byte units
  float fx[3], fy[3];
};
// The nw texel is clamped to R-2, so that all four taps always exist at fixed offsets (+128 B, +one
// row): at the far edge the fraction becomes 1 instead of 0 on the next cell, the interpolated value
// is the same bit for bit (0 * finite + 1 * v), and the serving lanes need two address computations
// per plane instead of four (instead of two "neighbour exists" flag bits per tap).
__device__ __forceinline__ void byte_taps(float gx, float gy, int R, uint32_t plane_units,
                                          uint32_t& o, float& fx, float& fy) {
  const float m = (float)(R - 1);
  float ix = (gx + 1.f) * 0.5f * m;
  float iy = (gy + 1.f) * 0.5f * m;
  ix = fminf(m, fmaxf(ix, 0.f));
  iy = fminf(m, fmaxf(iy, 0.f));
  const float x0 = fminf(floorf(ix), m - 1.f), y0 = fminf(floorf(iy), m - 1.f);
  fx = ix - x0;
  fy = iy - y0;
  o = plane_units + (uint32_t)((int)y0 * R + (int)x0) * 8u;
}
// base + 16 * off as ONE IMAD.WIDE.U32 (a plain 64-bit pointer add costs two)
__device__ __forceinline__ const float4* texel_ptr(const unsigned char* base, uint32_t off16) {
  uint64_t r;
  asm("mad.wide.u32 %0, %1, 16, %2;" : "=l"(r) : "r"(off16), "l"(base));
  return reinterpret_cast<const float4*>(r);
}
__device__ __forceinline__ float4 ldg_nc_volatile_next(const float4* p) {  // the texel one to the east
  float4 r;
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4+128];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
// How gather_to_tiles_lean stores the features of a point (a row of the tile):
//   kTf32Pair  a TF32 hi/lo PAIR in two [128 rows][32 fp32] SWIZZLE_128B tiles, the shared-memory
//              A operands of a 3xTF32 layer 1;
//   kBf16Pair  a bf16 hi/lo PAIR in two [128 rows][32 bf16] SWIZZLE_64B tiles (64-byte rows): half
//              the bytes, and a layout that is both the K-major A operand of a bf16 layer-1 MMA and
//              -- rows = K -- an MN-major B operand (nfi_wgrad_pipe.cuh);
//   kFp32      the fp32 features once, in one SWIZZLE_128B tile laid out like the kTf32Pair hi tile
//              (`a_lo` unused): the consumer loads its A fragments and splits them in registers
//              (nfi_forward_pipe.cuh).
enum class TileStore { kTf32Pair, kBf16Pair, kFp32 };
template <TileStore MODE = TileStore::kTf32Pair>
__device__ __forceinline__ void gather_to_tiles_lean(const unsigned char* __restrict__ planes_b,
                                                     int R, const ByteTaps& tp,
                                                     unsigned char* a_hi, unsigned char* a_lo,
                                                     int row0, int lane) {
  const int q = lane >> 3, k = lane & 7;
  const uint32_t row_units = (uint32_t)R * 8u;
#pragma unroll 1
  for (int g = 0; g < 8; ++g) {
    const int src = 4 * g + q;
    float4 v[12];
    float fx[3], fy[3];
#pragma unroll
    for (int pl = 0; pl < 3; ++pl) {
      const uint32_t o = __shfl_sync(kFull, tp.o[pl], src);
      fx[pl] = __shfl_sync(kFull, tp.fx[pl], src);
      fy[pl] = __shfl_sync(kFull, tp.fy[pl], src);
      const uint32_t a00 = o | (uint32_t)k;
      const float4* p0 = texel_ptr(planes_b, a00);
      const float4* p1 = texel_ptr(planes_b, a00 + row_units);
      v[4 * pl + 0] = ldg_nc_volatile(p0);
      v[4 * pl + 1] = ldg_nc_volatile_next(p0);
      v[4 * pl + 2] = ldg_nc_volatile(p1);
      v[4 * pl + 3] = ldg_nc_volatile_next(p1);
    }
    float2 lo = make_float2(0.f, 0.f), hi = make_float2(0.f, 0.f);
#pragma unroll
    for (int pl = 0; pl < 3; ++pl) {
      const float gx0 = 1.f - fx[pl], gy0 = 1.f - fy[pl];
      const float w[4] = {gx0 * gy0, fx[pl] * gy0, gx0 * fy[pl], fx[pl] * fy[pl]};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 x = v[4 * pl + j];
        lo = ffma2(make_float2(x.x, x.y), make_float2(w[j], w[j]), lo);
        hi = ffma2(make_float2(x.z, x.w), make_float2(w[j], w[j]), hi);
      }
    }
    const float third = 0.33333334f;
    const float4 f = make_float4(lo.x * third, lo.y * third, hi.x * third, hi.y * third);
    if constexpr (MODE == TileStore::kFp32) {
      *reinterpret_cast<float4*>(a_hi + tc::sw128_offset(row0 + src, k)) = f;
    } else if constexpr (MODE == TileStore::kBf16Pair) {
      uint2 h, l;
      asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h.x) : "f"(f.y), "f"(f.x));
      asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(h.y) : "f"(f.w), "f"(f.z));
      const float rx = f.x - __uint_as_float(h.x << 16), ry = f.y - __uint_as_float(h.x & 0xFFFF0000u);
      const float rz = f.z - __uint_as_float(h.y << 16), rw = f.w - __uint_as_float(h.y & 0xFFFF0000u);
      asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(l.x) : "f"(ry), "f"(rx));
      asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(l.y) : "f"(rw), "f"(rz));
      const uint32_t offs = tc::sw64_offset(row0 + src, k >> 1) + (k & 1) * 8;
      *reinterpret_cast<uint2*>(a_hi + offs) = h;
      *reinterpret_cast<uint2*>(a_lo + offs) = l;
    } else {
      const float4 fh = make_float4(tc::tf32_hi(f.x), tc::tf32_hi(f.y), tc::tf32_hi(f.z),
                                    tc::tf32_hi(f.w));
      const float4 fl = make_float4(f.x - fh.x, f.y - fh.y, f.z - fh.z, f.w - fh.w);
      const uint32_t offs = tc::sw128_offset(row0 + src, k);
      *reinterpret_cast<float4*>(a_hi + offs) = fh;
      *reinterpret_cast<float4*>(a_lo + offs) = fl;
    }
  }
}

struct TcShared {
  unsigned char* base;   // 1024-aligned
  const float* b1;
  const float* b2;
  float* pal;
  uint64_t* bars;        // [0] weights
};

__device__ __forceinline__ TcShared tc_shared_map(unsigned char* raw) {
  TcShared s;
  s.base = raw;  // declared __align__(1024); checked in tc_prologue
  s.b1 = reinterpret_cast<const float*>(raw + kWiB1);
  s.b2 = reinterpret_cast<const float*>(raw + kWiB2);
  s.pal = reinterpret_cast<float*>(raw + kSmPal);
  s.bars = reinterpret_cast<uint64_t*>(raw + kSmBars);
  return s;
}

// per-thread view of its tile group
struct TcGroup {
  int g, gt, wig;
  unsigned char* a_hi;   // A_hi tile
  unsigned char* a_lo;   // A_lo tile
  float* out;            // decoder outputs, [128][kOutLd]
  uint64_t dsc_a, dsc_w1_hi, dsc_w1_lo, dsc_w2_hi, dsc_w2_lo;  // wgmma descriptor bases
};

__device__ __forceinline__ TcGroup tc_group(const TcShared& sm, int tid) {
  TcGroup q;
  // warp-uniform by construction AND known to the compiler as such (shfl from lane 0):
  // lets ptxas keep the wgmma operands in uniform registers
  q.g = __shfl_sync(kFull, tid >> 7, 0);
  q.gt = tid & 127;
  q.wig = __shfl_sync(kFull, q.gt >> 5, 0);
  q.a_hi = sm.base + kSmA + q.g * kSmAGroup;
  q.a_lo = q.a_hi + 16384;
  q.out = reinterpret_cast<float*>(sm.base + kSmOut) + q.g * kThreads * kOutLd;
  const uint32_t base_s = tc::smem_u32(sm.base);
  q.dsc_a = tc::gmma_desc_sw128(base_s + kSmA + q.g * kSmAGroup);
  q.dsc_w1_hi = tc::gmma_desc_sw128(base_s + kWiW1Hi);
  q.dsc_w1_lo = tc::gmma_desc_sw128(base_s + kWiW1Lo);
  q.dsc_w2_hi = tc::gmma_desc_sw128(base_s + kWiW2Hi);
  q.dsc_w2_lo = tc::gmma_desc_sw128(base_s + kWiW2Lo);
  return q;
}

// The decoder on one 128-point tile whose features already sit (hi/lo split)
// in the group's A tiles.  Both linear layers run on the tensor core, one
// 64-row half of the tile after the other (the group is one warpgroup):
//   layer 1    : D1 = A * W1^T                      (12 x wgmma, N = 64, registers)
//   epilogue 1 : h = softplus(D1 + b1) -> H_hi / H_lo register A fragments
//   layer 2    : D2 = H * W2^T                      (24 x wgmma, N = 16)
//   epilogue 2 : D2 -> the group's output tile; out = D2 + b2 of this thread's row
template <int NOUT_PAD>
__device__ __forceinline__ void tile_mlp(const TcGroup& q, const TcShared& sm,
                                         float (&out)[NOUT_PAD]) {
  const int lane = q.gt & 31;
  tc::fence_async_smem();
  tc::bar_sync(1 + q.g, kThreads);  // A tiles complete, previous outputs consumed
#pragma unroll 1
  for (int mb = 0; mb < 2; ++mb) {
    float d[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) d[i] = 0.f;
    tc::wgmma_fence();
    tc::layer1_mb(d, q.dsc_a + mb * (8192 >> 4), q.dsc_a + ((16384 + mb * 8192) >> 4), q.dsc_w1_hi,
                  q.dsc_w1_lo);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::reg_fence(d);
    uint32_t hi[8][4], lo[8][4];
    tc::softplus_frag<false>(d, sm.b1, lane & 3, hi, lo);
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = 0.f;
    tc::wgmma_fence();
    tc::layer2_mb(o, hi, lo, q.dsc_w2_hi, q.dsc_w2_lo);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::reg_fence(o);
    tc::store_frag_rows(o, q.out + 64 * mb * kOutLd, kOutLd, q.wig, lane);
  }
  tc::bar_sync(1 + q.g, kThreads);
  const float* row = q.out + q.gt * kOutLd;
#pragma unroll
  for (int o = 0; o < NOUT_PAD; ++o) out[o] = row[o] + sm.b2[o];
}

// common prologue: barrier, weight image via TMA bulk copy
__device__ __forceinline__ void tc_prologue(const TcShared& sm, const unsigned char* wimg,
                                            int tid) {
  if (tid == 0) {
    if (tc::smem_u32(sm.base) & 1023u) __trap();  // SWIZZLE_128B tiles need 1024-byte alignment
    tc::mbar_init(&sm.bars[0], 1);
    tc::fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    tc::mbar_expect_tx(&sm.bars[0], kWiBytes);
    tc::tma_bulk_g2s(sm.base, wimg, kWiBytes, &sm.bars[0]);
  }
  tc::mbar_wait(&sm.bars[0], 0);
}

// ---------------------------------------------------------------------------
// Stand-alone decoder: features [N,32] -> decoder outputs [N,nout]
// (TriplanarDecoder.net, models/generator.py:294-299,329-331).  Same tiles,
// descriptors, barriers and epilogue as the render kernel.
// ---------------------------------------------------------------------------
template <int NOUT_PAD>
__global__ void __launch_bounds__(kTcThreads, 1)
decoder_forward_tc(const float* __restrict__ feats, long long n_points, int nout,
                   const unsigned char* __restrict__ wimg, float* __restrict__ outp) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const TcShared sm = tc_shared_map(smem_raw);
  const int tid = threadIdx.x;
  tc_prologue(sm, wimg, tid);
  const TcGroup q = tc_group(sm, tid);
  const long long n_tiles = (n_points + 127) / 128;
  for (long long tile = (long long)blockIdx.x * kGroups + q.g; tile < n_tiles;
       tile += (long long)gridDim.x * kGroups) {
    const long long row = tile * 128 + q.gt;  // thread gt stages row gt: 8 x 16 bytes
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row < n_points) f = *reinterpret_cast<const float4*>(feats + row * kC + 4 * c);
      const float4 fh = make_float4(tc::tf32_hi(f.x), tc::tf32_hi(f.y), tc::tf32_hi(f.z),
                                    tc::tf32_hi(f.w));
      const float4 fl = make_float4(f.x - fh.x, f.y - fh.y, f.z - fh.z, f.w - fh.w);
      const uint32_t off = tc::sw128_offset(q.gt, c);
      *reinterpret_cast<float4*>(q.a_hi + off) = fh;
      *reinterpret_cast<float4*>(q.a_lo + off) = fl;
    }
    float out[NOUT_PAD];
    tile_mlp<NOUT_PAD>(q, sm, out);
    if (row < n_points)
      for (int o = 0; o < NOUT_PAD; ++o)
        if (o < nout) outp[row * nout + o] = out[o];
  }
}

// ---------------------------------------------------------------------------
// render, tensor-core variant.  EXTRA: 0 none, 1 coords.
// ---------------------------------------------------------------------------
template <int NOUT_PAD, int EXTRA, bool FINE>
__global__ void __launch_bounds__(kTcThreads, 1)
render_forward_tc(const nfi_render_params p, const unsigned char* __restrict__ wimg,
                  float* __restrict__ scratch) {
  constexpr int NE = (EXTRA == 1) ? 3 : 0;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const TcShared sm = tc_shared_map(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31;
  const int S = p.num_samples;
  tc_prologue(sm, wimg, tid);
  const TcGroup q = tc_group(sm, tid);
  const int g = q.g, gt = q.gt, wig = q.wig;

  // CTA -> 2x2 block of 16x8 tiles of one image
  const int tiles_x = (p.width + kTileW - 1) / kTileW;
  const int tiles_y = (p.height + kTileH - 1) / kTileH;
  const int ctx_n = (tiles_x + 1) / 2, cty_n = (tiles_y + 1) / 2;
  const int cta = blockIdx.x;
  const int b = cta / (ctx_n * cty_n);
  const int crem = cta % (ctx_n * cty_n);
  const int tile_x = 2 * (crem % ctx_n) + (g & 1);
  const int tile_y = 2 * (crem / ctx_n) + (g >> 1);
  const bool group_active = (tile_x < tiles_x) && (tile_y < tiles_y);

  if (tid < 48)
    sm.pal[tid] = (p.n_attention > 0 && tid < p.n_attention * 3)
                      ? p.palette[(size_t)b * p.n_attention * 3 + tid]
                      : 0.f;
  __syncthreads();

  if (group_active) {
    int px, py;
    tile_pixel(tile_x, tile_y, wig, lane, px, py);
    const bool valid = (px < p.width) && (py < p.height);
    px = min(px, p.width - 1);
    py = min(py, p.height - 1);
    const size_t ray = ((size_t)b * p.height + py) * p.width + px;
    Ray r;
    setup_ray(p, b, py, px, r);
    FieldConst fc;
    fc.A = p.n_attention;
    fc.use_sdf = p.use_sdf;
    fc.inv_beta = p.use_sdf ? 1.f / p.beta[0] : 0.f;
    fc.inv_alpha = p.use_sdf ? 1.f / p.alpha[0] : 0.f;
    const float inv_range = 1.f / p.scene_range;
    const int R = p.plane_res;
    const float* planes_b = p.planes + (size_t)b * 3 * R * R * kC;
    const bool explicit_noise = (p.noise_mode == NFI_NOISE_EXPLICIT);

    unsigned char* a_hi = q.a_hi;
    unsigned char* a_lo = q.a_lo;

    const size_t group_slot = (size_t)blockIdx.x * kGroups + g;
    float* slab = scratch + group_slot * tc_scratch_floats_per_group(S);
    float4* sc_srgb = reinterpret_cast<float4*>(slab);
    float* sc_t = slab + (size_t)4 * S * kThreads;
    float* sc_w = sc_t + (size_t)S * kThreads;
    float* sc_zf = sc_w + (size_t)S * kThreads;

    Compositor<NE, true> comp;
    comp.init();

    auto eval = [&](float t, float& sigma, float& cr, float& cg, float& cb, float* ex) {
      const float wx = r.ox + r.dx * t, wy = r.oy + r.dy * t, wz = r.oz + r.dz * t;
      const float x0 = wx * inv_range, x1 = wy * inv_range, x2 = wz * inv_range;
      const float keep =
          (fabsf(x0) > 1.f || fabsf(x1) > 1.f || fabsf(x2) > 1.f) ? 0.f : 1.f;
      PackedTaps tp;
      pack_taps(x0, x1, R, tp.o[0], tp.fx[0], tp.fy[0]);
      pack_taps(x0, x2, R, tp.o[1], tp.fx[1], tp.fy[1]);
      pack_taps(x1, x2, R, tp.o[2], tp.fx[2], tp.fy[2]);
      gather_to_tiles_deep(planes_b, R, tp, a_hi, a_lo, 32 * wig, lane);
      float out[NOUT_PAD];
      tile_mlp<NOUT_PAD>(q, sm, out);
      float probs[NOUT_PAD];
      field_head<NOUT_PAD, true>(out, fc, sm.pal, keep, sigma, cr, cg, cb, probs);
      if (EXTRA == 1) {
        ex[0] = wx;
        ex[1] = wy;
        ex[2] = wz;
      }
    };

    // ---------------- coarse pass ----------------
    float wT = 1.f, prev_t = 0.f, prev_s = 0.f;
    const float span = r.tfar - r.tnear;
    for (int s = 0; s < S; ++s) {
      float t = lerp_torch(r.tnear, r.tfar, (float)s / (float)S);
      if (explicit_noise) t = t + p.noise_t[ray * S + s] * (span / (float)S);
      float sigma, cr, cg, cb;
      float ex[NE > 0 ? NE : 1];
      eval(t, sigma, cr, cg, cb, ex);
      if (FINE) {
        sc_srgb[s * kThreads + gt] = make_float4(sigma, cr, cg, cb);
        sc_t[s * kThreads + gt] = t;
        if (s > 0) {
          const float delta = (t - prev_t) * r.dn;
          const float a = 1.f - expf(-prev_s * delta);
          sc_w[(s - 1) * kThreads + gt] = a * wT;
          wT = wT * ((1.f - a) + 1e-10f);
        }
        prev_t = t;
        prev_s = sigma;
      } else {
        comp.push(t, sigma, cr, cg, cb, ex, r.dn);
      }
    }

    if (FINE) {
      sc_w[(S - 1) * kThreads + gt] = 0.f;
      // the A tiles are idle until pass 2: use them as S x 128 float columns
      float* col = reinterpret_cast<float*>(a_hi) + gt;
      // smoothed pdf (run.py:266-272, lib/nerf_utils.py:189-192): first the sum
      float sum = 0.f;
      {
        float wa = sc_w[gt], wb = sc_w[kThreads + gt], wc;
        for (int m = 0; m + 2 < S; ++m) {
          wc = sc_w[(m + 2) * kThreads + gt];
          sum += ((fmaxf(wa, wb) + fmaxf(wb, wc)) * 0.5f + 0.01f) + 1e-5f;
          wa = wb;
          wb = wc;
        }
      }
      // the S uniforms, ascending (thread-private column: bank = thread)
      if (explicit_noise) {
        for (int k = 0; k < S; ++k) {
          const float u = p.noise_u[ray * S + k];
          int i = k - 1;
          while (i >= 0 && col[i * kThreads] > u) {
            col[(i + 1) * kThreads] = col[i * kThreads];
            --i;
          }
          col[(i + 1) * kThreads] = u;
        }
      } else {
        for (int k = 0; k < S; ++k) col[k * kThreads] = linspace01(k, S);
      }
      // inverse CDF: walk the CDF bins once, consuming the sorted uniforms
      {
        int k = 0;
        float c_prev = 0.f;
        float wa = sc_w[gt], wb = sc_w[kThreads + gt], wc;
        float t_lo = sc_t[gt], t_mid = sc_t[kThreads + gt];
        float z0 = 0.5f * (t_mid + t_lo);  // bins[0]
        for (int i = 1; i + 1 < S; ++i) {  // cdf[i], i = 1 .. S-2
          wc = sc_w[(i + 1) * kThreads + gt];
          const float pw = ((fmaxf(wa, wb) + fmaxf(wb, wc)) * 0.5f + 0.01f) + 1e-5f;
          wa = wb;
          wb = wc;
          const float c_i = c_prev + pw / sum;
          const float t_hi = sc_t[(i + 1) * kThreads + gt];
          const float z1 = 0.5f * (t_hi + t_mid);  // bins[i]
          float den = c_i - c_prev;
          if (den < 1e-5f) den = 1.f;
          while (k < S) {
            const float u = col[k * kThreads];
            if (!(u < c_i)) break;
            col[k * kThreads] = z0 + (u - c_prev) / den * (z1 - z0);
            ++k;
          }
          c_prev = c_i;
          t_mid = t_hi;
          z0 = z1;
        }
        while (k < S) {  // u >= cdf[S-2]: both neighbours are the last bin
          col[k * kThreads] = z0;
          ++k;
        }
      }
      if (p.z_fine != nullptr && valid)
        for (int k = 0; k < S; ++k) p.z_fine[ray * S + k] = col[k * kThreads];
      // park the sorted fine depths next to the coarse samples (coalesced)
      for (int k = 0; k < S; ++k) sc_zf[k * kThreads + gt] = col[k * kThreads];
      __syncwarp();
      tc::bar_sync(1 + g, kThreads);  // columns are dead; A tiles may be rewritten

      // ------- fine pass + sorted merge + compositing -------
      int c = 0;
      float ct = sc_t[gt];
      for (int k = 0; k < S; ++k) {
        const float z = sc_zf[k * kThreads + gt];
        float sigma, cr, cg, cb;
        float ex[NE > 0 ? NE : 1];
        eval(z, sigma, cr, cg, cb, ex);
        while (c < S && ct <= z) {
          const float4 q = sc_srgb[c * kThreads + gt];
          float ce[NE > 0 ? NE : 1];
          if (EXTRA == 1) {
            ce[0] = r.ox + r.dx * ct;
            ce[1] = r.oy + r.dy * ct;
            ce[2] = r.oz + r.dz * ct;
          }
          comp.push(ct, q.x, q.y, q.z, q.w, ce, r.dn);
          ++c;
          ct = (c < S) ? sc_t[c * kThreads + gt] : 0.f;
        }
        comp.push(z, sigma, cr, cg, cb, ex, r.dn);
      }
      while (c < S) {
        const float4 q = sc_srgb[c * kThreads + gt];
        float ce[NE > 0 ? NE : 1];
        if (EXTRA == 1) {
          ce[0] = r.ox + r.dx * ct;
          ce[1] = r.oy + r.dy * ct;
          ce[2] = r.oz + r.dz * ct;
        }
        comp.push(ct, q.x, q.y, q.z, q.w, ce, r.dn);
        ++c;
        ct = (c < S) ? sc_t[c * kThreads + gt] : 0.f;
      }
    }

    if (valid) {
      float bg = 0.f;
      if (p.white_background) bg = 1.f - comp.am;
      p.rgb[ray * 3 + 0] = comp.ar + bg;
      p.rgb[ray * 3 + 1] = comp.ag + bg;
      p.rgb[ray * 3 + 2] = comp.ab + bg;
      p.depth[ray] = comp.ad;
      p.mask[ray] = comp.am;
      if (EXTRA == 1 && p.extra != nullptr)
        for (int a = 0; a < 3; ++a) p.extra[ray * 3 + a] = comp.ae[a];
    }
  }
}

}  // namespace nfi
