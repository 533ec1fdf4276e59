// Tensor-core building blocks of the decoder, shared by the pipelined kernels (nfi_*_pipe.cuh) and
// the stand-alone decoder behind nfi_decoder_forward:
//
//   weight image   the decoder weights pre-split into TF32 hi / lo parts and pre-swizzled as wgmma
//                  B operands, plus the biases (prep_weight_image, nfi_weight_image.cuh); a kernel brings it into shared
//                  memory with ONE TMA bulk copy per CTA;
//   plane gather   gather_to_tiles_lean: a warp's 32 points gathered cooperatively (8 lanes x
//                  float4 = one 128-byte channel-last texel per tap), interpolated and written
//                  straight into a shared-memory operand tile -- features never exist anywhere else;
//   decoder tile   decoder_forward_tc: CTA = 512 threads = 4 tile groups of 128 threads (one
//                  warpgroup each); a group stages 128 feature rows as TF32 hi / lo A tiles and runs
//                  both decoder layers on wgmma (3xTF32), one 64-row half of the tile after the
//                  other (tile_mlp).
#pragma once
#include "nfi_common.cuh"
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
static_assert(kWiBytes <= kFwdImageSlot, "weight image larger than the workspace header");
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

__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

__device__ __forceinline__ float4 ldg_nc_volatile(const float4* p) {
  float4 r;  // volatile: the 12 loads of a point group must issue back-to-back, before any use
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

// ---------------------------------------------------------------------------
// Lean gather.  The owner lane of a point pre-multiplies its three nw-texel
// offsets into offsets from the image's plane base in 16-byte units (plane index
// and the 8 units of a texel included), so the serving lanes only OR in their
// channel quad and widen (one IMAD.WIDE.U32 per address: x16 + base).  Per point
// group (4 points x 8 lanes) the 12 texel loads are ISSUED TOGETHER, then
// interpolated: a structure that interleaves loads and FFMA2s leaves only ~4
// loads in flight per warp and serialises ~24 L2 round trips per step.
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
// (TriplanarDecoder.net, models/generator.py:294-299,329-331).  Each tile group
// strides over the 128-point tiles; its 128 threads stage one feature row each.
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

}  // namespace nfi
