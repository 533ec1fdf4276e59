// Forward render kernel, pipelined tensor-core variant (NFI_MLP_TC_PIPE, the default).
//
// A 3xTF32 decoder on wgmma (weight image and plane gather from nfi_forward_tc.cuh), thread =
// ray for everything per-ray.  The per-step chain
//     gather -> MMA1 -> softplus/split -> MMA2 -> density/colour/composite
// is cut so that NO resource is held across more than one link of it, and every
// role only ever does its own kind of work:
//
//   persistent CTA (one per SM), one 16x8-pixel tile (128 rays) in flight:
//     warpgroup 0   ACTIVATION  loads the stage's features as register A fragments, splits
//                   them into TF32 hi / lo and issues both decoder layers (wgmma, accumulators
//                   in its registers, one 64-row half of the tile after the other): D1 ->
//                   softplus -> H_hi / H_lo register A fragments -> D2 -> D2 slot in shared memory
//     warpgroup 1   SHADING     thread = ray: D2 -> density / colour -> coarse
//                   weights or sorted merge + compositing (latency-bound chains);
//                   the two groups put two independent instruction streams on
//                   every SM sub-partition
//     warpgroups 2+ P PRODUCER sets of 4 warps; set q gathers the steps n = q (mod P)
//                   into A stage n mod (P+1) (fp32 features, 16 KB, SWIZZLE_128B)
//
//   stage   : producers --full[q]--> activation --a_free[q]--> producers
//             (a stage is released as soon as the activation group has loaded its
//             fragments, before any tensor work; the hidden activations never come
//             back to shared memory)
//   L1      : the stages are kept small because every byte of shared memory is taken from
//             the L1 that serves the plane gather (run_fwd sets the carve-out)
//   D2 slot : three [128 x 20] fp32 slots: activation --d2_full--> shading --slot_free-->
//             activation
//   softplus: ln2 * (max(x', 0) + lg2(1 + 2^-|x'|)) with x' = x log2 e: two MUFU ops (ex2, lg2)
//             per hidden unit; log2(e) is folded into W1/b1 by prep_weight_image;
//   view    : the VD instantiation (--use_viewdir) puts a third layer behind the decoder in the
//             activation warpgroup (decoder_layers23_vd below); every other role is unchanged
//   resample: the S uniforms of a ray are sorted by a bitonic network across the
//             warp (2 per lane) and pushed through the inverse CDF with shuffle
//             binary searches: one warp-pass per ray instead of a serial per-thread
//             walk (run.py:259-281, lib/nerf_utils.py:183-222).
#pragma once
#include <type_traits>

#include "nfi_forward.cuh"
#include "nfi_forward_tc.cuh"

namespace nfi {

// back-off between mbarrier polls of the per-step hand-offs (0 = hardware-suspended try_wait only)
#ifndef NFI_WAIT_NS
#define NFI_WAIT_NS 0
#endif
#define NFI_STEP_WAIT(bar, par) tc::mbar_wait_backoff<NFI_WAIT_NS>(bar, par)

// ------------------------------------------------------------------ small helpers
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tc::smem_u32(bar)) : "memory");
}

__device__ __forceinline__ float ld_relaxed(const float* p) {
  float v;
  asm volatile("ld.relaxed.cta.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n.reg .pred p;\nelect.sync _|p, 0xffffffff;\nselp.u32 %0, 1, 0, p;\n}\n"
      : "=r"(pred));
  return pred != 0;
}

struct TileCoord {
  int b, tile_x, tile_y;
};

__device__ __forceinline__ TileCoord tile_coord(int tile, int tiles_x, int tiles_y) {
  TileCoord c;
  const int per_img = tiles_x * tiles_y;
  c.b = tile / per_img;
  const int r = tile % per_img;
  // 2x2 blocks of tiles are consecutive: the two groups of a CTA (and the next
  // CTA) work on neighbouring tiles of the same image -> shared texels in L1/L2
  const int bx = (tiles_x + 1) / 2;
  const int blk = r / 4, in = r % 4;
  int tx = 2 * (blk % bx) + (in & 1), ty = 2 * (blk / bx) + (in >> 1);
  if ((tiles_x & 1) || (tiles_y & 1)) {  // odd tile grids: plain row-major order
    tx = r % tiles_x;
    ty = r / tiles_x;
  }
  c.tile_x = tx;
  c.tile_y = ty;
  return c;
}

constexpr int kPipeSlots = 3;
constexpr int kPipeStageBytes = 32768;
constexpr int kFwdStageBytes = 16384;  // fp32 features of 128 points (the TF32 split is done in registers)
constexpr int kD2Ld = 20;  // floats per row of a D2 slot (80-byte rows: row reads are conflict-free)
constexpr int kD2SlotBytes = kThreads * kD2Ld * 4;

// scratch per CTA: the tc_scratch layout plus NES parked extras per coarse sample
__host__ __device__ inline size_t pipe_scratch_floats(int S, int nes) {
  return tc_scratch_floats_per_group(S) + (size_t)S * kThreads * nes;
}

// view features of a tile plus b2[1..32], in the layer-2 accumulator's fragment order (VD only)
constexpr int kViewTileBytes = kThreads * NFI_VIEW_FEATURES * 4;

// VD: the view-direction-conditioned instantiation (a larger weight image, nfi_layout.h, and the
// tile's view features); the offsets of the plain kernel do not depend on it.
template <int P, bool VD = false>
struct PipeCfg {
  static constexpr int kThreadsTotal = 256 + 128 * P;
  static constexpr int kStages = P + 1;  // one spare: a set never waits for its own MMA
  static constexpr int kSmA = VD ? 41984 : 25600;
  static constexpr int kSmD2 = kSmA + kStages * kFwdStageBytes;
  static constexpr int kSmView = kSmD2 + kPipeSlots * kD2SlotBytes;
  static constexpr int kSmPal = kSmView + (VD ? kViewTileBytes : 0);
  static constexpr int kSmFrac = kSmPal + 48 * 4;  // s / S for s < 128 (one IEEE division each)
  static constexpr int kSmBars = kSmFrac + 128 * 4;
  // full[P+1], a_free[P+1], d2_full[3], slot_free[3], cw_ready, zf_ready, weights
  static constexpr int kNumBars = 2 * kStages + 2 * kPipeSlots + 3;
  static constexpr int kSmBytes = kSmBars + kNumBars * 8;
  // setmaxnreg moves registers inside the CTA's launch allocation (threads x launch regs):
  //   P = 3: 640 x 96 = 61440 = 128 x (136 + 80) + 384 x 88 (12 texel loads in flight per
  //   producer warp: 48 data registers + 64-bit addresses + taps; the activation group holds a
  //   64 x 64 accumulator block and its hi / lo split, plus the 16 feature values of the second
  //   64-row half).
  static constexpr int kActRegs = 136;
  static constexpr int kShadeRegs = 80;
  static constexpr int kProducerRegs = 88;
};

// this kernel's weight image has log2(e) folded into layer 1 (the softplus works
// on x' = x log2 e) and padded colour logits pushed to -1e30 (softmax needs no mask)
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr float kPadLogit = -1e30f;

// Second half of the decoder for one 64-row block, issued by the whole warpgroup: softplus on the
// layer-1 accumulator registers, layer 2 with H as register A fragments (24 wgmma), D2 rows to `d2`.
__device__ __forceinline__ void decoder_layer2(const float (&d)[32], uint64_t w2_hi, uint64_t w2_lo,
                                               const float* __restrict__ b1, float* d2, int warp,
                                               int lane) {
  uint32_t hi[8][4], lo[8][4];
  tc::softplus_frag<true>(d, b1, lane & 3, hi, lo);
  float o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = 0.f;
  tc::wgmma_fence();
  tc::layer2_mb(o, hi, lo, w2_hi, w2_lo);
  tc::wgmma_commit();
  tc::wgmma_wait<0>();
  tc::reg_fence(o);
  tc::store_frag_rows(o, d2, kD2Ld, warp, lane);
}

// The decoder of one 128-point step, issued by the whole (activation) warpgroup: per 64-row
// half, layer 1 from a TF32 hi / lo A stage in shared memory (3xTF32, 12 wgmma), then
// decoder_layer2.  `on_stage_read` runs once layer 1 of both halves has completed (the stage may
// be refilled); D2 goes to `d2` ([128][kD2Ld]).
template <typename F>
__device__ __forceinline__ void decoder_step(uint64_t dsc_a, uint64_t w1_hi, uint64_t w1_lo,
                                             uint64_t w2_hi, uint64_t w2_lo,
                                             const float* __restrict__ b1, float* d2, int warp,
                                             int lane, F&& on_stage_read) {
#pragma unroll 1
  for (int mb = 0; mb < 2; ++mb) {
    float d[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) d[i] = 0.f;
    tc::wgmma_fence();
    tc::layer1_mb(d, dsc_a + mb * (8192 >> 4), dsc_a + ((16384 + mb * 8192) >> 4), w1_hi, w1_lo);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::reg_fence(d);
    if (mb == 1) on_stage_read();
    decoder_layer2(d, w2_hi, w2_lo, b1, d2 + 64 * mb * kD2Ld, warp, lane);
  }
}

// The same decoder from an fp32 feature stage ([128 x 32], SWIZZLE_128B): the warpgroup loads the
// A fragments of both halves, `on_stage_read` runs (the stage may be refilled before any tensor
// work on it), and each half is split into TF32 hi / lo in registers exactly as the producers of
// a hi / lo stage would split it, so layer 1 sees the same operands as decoder_step.
template <typename F>
__device__ __forceinline__ void decoder_step_fp32(const unsigned char* stage, uint64_t w1_hi,
                                                  uint64_t w1_lo, uint64_t w2_hi, uint64_t w2_lo,
                                                  const float* __restrict__ b1, float* d2, int warp,
                                                  int lane, F&& on_stage_read) {
  float fa[4][4], fb[4][4];  // the features of the current half, of the second half
  tc::load_afrag_sw128(fa, stage, 0, warp, lane);
  tc::load_afrag_sw128(fb, stage, 64, warp, lane);
  on_stage_read();
#pragma unroll 1
  for (int mb = 0; mb < 2; ++mb) {
    uint32_t a_hi[4][4], a_lo[4][4];
#pragma unroll
    for (int kb = 0; kb < 4; ++kb)
#pragma unroll
      for (int s = 0; s < 4; ++s) tc::put_split(a_hi, a_lo, kb, s, fa[kb][s]);
    float d[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) d[i] = 0.f;
    tc::wgmma_fence();
    tc::layer1_mb_rs(d, a_hi, a_lo, w1_hi, w1_lo);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::reg_fence(d);
    decoder_layer2(d, w2_hi, w2_lo, b1, d2 + 64 * mb * kD2Ld, warp, lane);
#pragma unroll
    for (int kb = 0; kb < 4; ++kb)
#pragma unroll
      for (int s = 0; s < 4; ++s) fa[kb][s] = fb[kb][s];
  }
}

// ------------------------------------------------------------------ view-direction conditioning
// (--use_viewdir, models/generator.py:189-253,662-663): layer 2 emits the distance and 32
// features, and the colour logits are W3 . leaky_relu(view_features[ray] + features, 0.2) + b3.
// A step's row is a ray, so the view features are constant per row for the whole tile: the
// activation warpgroup keeps them (with b2[1..32] added) in shared memory in the order of its own
// layer-2 accumulator fragment -- float4 (mb, j) of thread gt holds rows g / g + 8 of 64-row block
// mb, columns 8j + 2t, 8j + 2t + 1 -- written and read by the same thread, so no barrier guards it.
__device__ __forceinline__ void fill_view_tile(const nfi_render_params& p, const TileCoord& tcd,
                                               const float* __restrict__ b2f, float4* vt, int wig,
                                               int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mb = 0; mb < 2; ++mb) {
    const float* src[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = 64 * mb + 16 * wig + g + 8 * h;
      int px, py;
      tile_pixel(tcd.tile_x, tcd.tile_y, row >> 5, row & 31, px, py);
      px = min(px, p.width - 1);  // rows outside the image: any finite value (masked later)
      py = min(py, p.height - 1);
      const size_t ray = ((size_t)tcd.b * p.height + py) * p.width + px;
      src[h] = p.view_features + ray * NFI_VIEW_FEATURES + 2 * t;
    }
#pragma unroll
    for (int j = 0; j < NFI_VIEW_FEATURES / 8; ++j) {
      const float2 a = __ldg(reinterpret_cast<const float2*>(src[0] + 8 * j));
      const float2 c = __ldg(reinterpret_cast<const float2*>(src[1] + 8 * j));
      const float2 bb = *reinterpret_cast<const float2*>(b2f + 8 * j + 2 * t);
      vt[(mb * 4 + j) * kThreads] = make_float4(a.x + bb.x, a.y + bb.y, c.x + bb.x, c.y + bb.y);
    }
  }
}

// Second half of the view-conditioned decoder for one 64-row block: softplus, layer 2 with N = 40
// (24 wgmma), leaky ReLU of features + view features on the accumulator registers, which become
// the register A fragments of layer 3 (12 wgmma), and the D2 row [distance, logits] to `d2`.
// Both accumulators start from zero and the fp32 terms (view features, biases, the distance) are
// added on the CUDA cores, as the plain kernel adds b2: the tensor core only sums products.
// Returns the leaky ReLU's branches: bit 4j + e set where element 4j + e of the accumulator took
// the 0.2 slope (the backward kernel replays them; the forward ignores the value).
__device__ __forceinline__ uint32_t decoder_layers23_vd(const float (&d)[32], uint64_t w2_hi,
                                                        uint64_t w2_lo, uint64_t w3_hi,
                                                        uint64_t w3_lo, const float* __restrict__ b1,
                                                        const float4* vt, float* d2, int warp,
                                                        int lane) {
  uint32_t hi[8][4], lo[8][4];
  tc::softplus_frag<true>(d, b1, lane & 3, hi, lo);
  float o[20];
#pragma unroll
  for (int i = 0; i < 20; ++i) o[i] = 0.f;
  tc::wgmma_fence();
  tc::layer2_vd_mb(o, hi, lo, w2_hi, w2_lo);
  tc::wgmma_commit();
  tc::wgmma_wait<0>();
  tc::reg_fence(o);
  uint32_t yhi[4][4], ylo[4][4];
  uint32_t neg = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 v = vt[j * kThreads];
    const float ve[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float z = o[4 * j + e] + ve[e];
      tc::put_split(yhi, ylo, j, tc::afrag_slot(e), z > 0.f ? z : z * 0.2f);
      neg |= (z > 0.f ? 0u : 1u) << (4 * j + e);
    }
  }
  float q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) q[i] = 0.f;
  tc::wgmma_fence();
  tc::layer3_vd_mb(q, yhi, ylo, w3_hi, w3_lo);
  tc::wgmma_commit();
  tc::wgmma_wait<0>();
  tc::reg_fence(q);
  // column 0 of layer 3 has zero weights; the thread that owns it (t = 0) also owns column 32
  // of layer 2, the distance, for the same two rows
  if ((lane & 3) == 0) {
    q[0] = o[16];
    q[2] = o[18];
  }
  tc::store_frag_rows(q, d2, kD2Ld, warp, lane);
  return neg;
}

// decoder_step_fp32 with the view-conditioned layers 2 and 3; `vt` = this thread's view tile.
// Returns the leaky ReLU branches of both halves (decoder_layers23_vd; half mb at bit 16 mb).
template <typename F>
__device__ __forceinline__ uint32_t decoder_step_vd(const unsigned char* stage, uint64_t w1_hi,
                                                uint64_t w1_lo, uint64_t w2_hi, uint64_t w2_lo,
                                                uint64_t w3_hi, uint64_t w3_lo,
                                                const float* __restrict__ b1, const float4* vt,
                                                float* d2, int warp, int lane, F&& on_stage_read) {
  float fa[4][4], fb[4][4];
  tc::load_afrag_sw128(fa, stage, 0, warp, lane);
  tc::load_afrag_sw128(fb, stage, 64, warp, lane);
  on_stage_read();
  uint32_t neg = 0;
#pragma unroll 1
  for (int mb = 0; mb < 2; ++mb) {
    uint32_t a_hi[4][4], a_lo[4][4];
#pragma unroll
    for (int kb = 0; kb < 4; ++kb)
#pragma unroll
      for (int s = 0; s < 4; ++s) tc::put_split(a_hi, a_lo, kb, s, fa[kb][s]);
    float d[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) d[i] = 0.f;
    tc::wgmma_fence();
    tc::layer1_mb_rs(d, a_hi, a_lo, w1_hi, w1_lo);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::reg_fence(d);
    neg |= decoder_layers23_vd(d, w2_hi, w2_lo, w3_hi, w3_lo, b1, vt + mb * 4 * kThreads,
                               d2 + 64 * mb * kD2Ld, warp, lane)
           << (16 * mb);
#pragma unroll
    for (int kb = 0; kb < 4; ++kb)
#pragma unroll
      for (int s = 0; s < 4; ++s) fa[kb][s] = fb[kb][s];
  }
  return neg;
}

__device__ __forceinline__ float ldcg(const float* p) {
  float v;
  asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}

// Density and colour from the decoder outputs, branch-free over the palette
// (padded logits arrive as -1e30, padded palette rows are zero).
// models/generator.py:625-679.
template <int NOUT_PAD>
__device__ __forceinline__ void field_head_fast(const float (&out)[NOUT_PAD], const FieldConst& fc,
                                                const float* __restrict__ pal, float keep,
                                                float& sigma, float& cr, float& cg, float& cb,
                                                float* probs = nullptr) {
  constexpr int NA = NOUT_PAD - 1;
  const float d = out[0];
  if (fc.use_sdf) {
    const float nd = -d;
    const float e = tc::ex2_approx(-fabsf(nd) * (fc.inv_beta * kLog2e));
    const float sg = (nd > 0.f) ? 1.f : ((nd < 0.f) ? -1.f : 0.f);
    const float cdf = 0.5f + 0.5f * sg * (1.f - e);
    sigma = fc.inv_alpha * (cdf * keep);
  } else {
    const float x = d - 1.f;
    sigma = (x > 20.f ? x : log1pf(expf(x))) * keep;
  }
  if (fc.A > 0) {
    // colour logits are in log2 units (prep_weight_image scales rows >= 1 of W2/b2)
    float m = out[1];
#pragma unroll
    for (int a = 1; a < NA; ++a) m = fmaxf(m, out[1 + a]);
    float pv[((3 * NA + 3) / 4) * 4];
#pragma unroll
    for (int i = 0; i < (3 * NA + 3) / 4; ++i) {
      const float4 t = *reinterpret_cast<const float4*>(pal + 4 * i);
      pv[4 * i] = t.x;
      pv[4 * i + 1] = t.y;
      pv[4 * i + 2] = t.z;
      pv[4 * i + 3] = t.w;
    }
    float s = 0.f, r = 0.f, g = 0.f, b = 0.f;
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      const float e = tc::ex2_approx(out[1 + a] - m);
      if (probs != nullptr) probs[a] = e;
      s += e;
      r = fmaf(e, pv[3 * a + 0], r);
      g = fmaf(e, pv[3 * a + 1], g);
      b = fmaf(e, pv[3 * a + 2], b);
    }
    const float inv = __fdividef(1.f, s);
    cr = r * inv;
    cg = g * inv;
    cb = b * inv;
    if (probs != nullptr) {
#pragma unroll
      for (int a = 0; a < NA; ++a) probs[a] *= inv;
    }
  } else {
    cr = sigmoid_fast(out[1]) * 2.004f - 1.002f;
    cg = sigmoid_fast(out[2]) * 2.004f - 1.002f;
    cb = sigmoid_fast(out[3]) * 2.004f - 1.002f;
  }
}

// ------------------------------------------------------------------ resampling
// Warp-per-ray importance resampling (run.py:266-281, lib/nerf_utils.py:183-222).
// Per-ray arrays of up to 32 N entries live N per lane: element e = 32 i + lane in v[i]
// (N = 2 for S <= 64, N = 4 for S <= 128).
template <int N>
struct LaneVec {
  float v[N];
};
// y_e = x_{e+1}; the element past the end is `pad`
template <int N>
__device__ __forceinline__ LaneVec<N> shift_down1(const LaneVec<N>& x, float pad, int lane) {
  LaneVec<N> y;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    const float a = __shfl_down_sync(kFull, x.v[i], 1);
    const float nxt0 = (i + 1 < N) ? __shfl_sync(kFull, x.v[(i + 1 < N) ? i + 1 : i], 0) : pad;
    y.v[i] = (lane == 31) ? nxt0 : a;
  }
  return y;
}
template <int N>
__device__ __forceinline__ float pick(const LaneVec<N>& x, int idx) {
  float r = __shfl_sync(kFull, x.v[0], idx & 31);
#pragma unroll
  for (int i = 1; i < N; ++i) {
    const float t = __shfl_sync(kFull, x.v[i], idx & 31);
    r = ((idx >> 5) == i) ? t : r;
  }
  return r;
}
// ascending bitonic sort of 32 N values
template <int N>
__device__ __forceinline__ void bitonic_sort(LaneVec<N>& x, int lane) {
#pragma unroll
  for (int k = 2; k <= 32 * N; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      if (j >= 32) {  // partner is another register of the same lane
        const int dj = j >> 5;
#pragma unroll
        for (int i = 0; i < N; ++i) {
          if ((i & dj) == 0) {
            const int ip = i | dj;
            const bool asc = (k >= 32 * N) ? true : (((32 * i) & k) == 0);
            const float lo = fminf(x.v[i], x.v[ip]), hi = fmaxf(x.v[i], x.v[ip]);
            x.v[i] = asc ? lo : hi;
            x.v[ip] = asc ? hi : lo;
          }
        }
      } else {
        const bool lower = (lane & j) == 0;
#pragma unroll
        for (int i = 0; i < N; ++i) {
          const float o = __shfl_xor_sync(kFull, x.v[i], j);
          // element index 32 i + lane: bit of k taken from the lane (k < 32) or from i
          const bool asc = (k >= 32 * N) ? true : (k < 32 ? ((lane & k) == 0) : (((32 * i) & k) == 0));
          x.v[i] = (lower == asc) ? fminf(x.v[i], o) : fmaxf(x.v[i], o);
        }
      }
    }
  }
}

// One ray.  w: coarse weights (elements >= S are don't-care), t: coarse depths,
// u: uniforms (padded with 2.0 beyond S; sorted inside unless `sorted`).  Returns
// the S fine depths in ascending order.
template <int N>
__device__ __forceinline__ LaneVec<N> resample_ray(const LaneVec<N>& w, const LaneVec<N>& t,
                                                   LaneVec<N> u, bool sorted, int S, int lane) {
  const float inf = __int_as_float(0x7f800000);
  // smoothed pdf p_m, m = 0 .. S-3  (run.py:266-272, + 1e-5 of sample_pdf)
  const LaneVec<N> w1 = shift_down1<N>(w, 0.f, lane);
  const LaneVec<N> w2 = shift_down1<N>(w1, 0.f, lane);
  LaneVec<N> q;
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    float pm = ((fmaxf(w.v[i], w1.v[i]) + fmaxf(w1.v[i], w2.v[i])) * 0.5f + 0.01f) + 1e-5f;
    if (32 * i + lane >= S - 2) pm = 0.f;
    q.v[i] = pm;
    sum += pm;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(kFull, sum, o);
  // inclusive scan of q_m = p_m / sum over the 32 N slots
#pragma unroll
  for (int i = 0; i < N; ++i) q.v[i] = q.v[i] / sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const float y = __shfl_up_sync(kFull, q.v[i], o);
      if (lane >= o) q.v[i] += y;
    }
  }
#pragma unroll
  for (int i = 1; i < N; ++i) q.v[i] += __shfl_sync(kFull, q.v[i - 1], 31);
  // cdf c_j, j = 0 .. S-2: c_0 = 0, c_j = scan_{j-1}; +inf beyond
  LaneVec<N> c;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    const float up = __shfl_up_sync(kFull, q.v[i], 1);
    const float prev31 = (i > 0) ? __shfl_sync(kFull, q.v[(i > 0) ? i - 1 : 0], 31) : 0.f;
    c.v[i] = (lane == 0) ? prev31 : up;
    if (32 * i + lane > S - 2) c.v[i] = inf;
  }
  // bins b_j = (t_j + t_{j+1}) / 2, j = 0 .. S-2
  const LaneVec<N> t1 = shift_down1<N>(t, 0.f, lane);
  LaneVec<N> bn;
#pragma unroll
  for (int i = 0; i < N; ++i) bn.v[i] = 0.5f * (t1.v[i] + t.v[i]);
  if (!sorted) bitonic_sort<N>(u, lane);
  LaneVec<N> z;
#pragma unroll
  for (int h = 0; h < N; ++h) {
    const float uu = u.v[h];
    int pos = 0;  // number of cdf entries <= u (searchsorted right=True)
#pragma unroll
    for (int s = 16 * N; s > 0; s >>= 1) {
      const float val = pick<N>(c, pos + s - 1);
      if (val <= uu) pos += s;
    }
    const int below = max(pos - 1, 0), above = min(pos, S - 2);
    const float c0 = pick<N>(c, below), c1 = pick<N>(c, above);
    const float b0 = pick<N>(bn, below), b1 = pick<N>(bn, above);
    float den = c1 - c0;
    if (den < 1e-5f) den = 1.f;
    z.v[h] = b0 + (uu - c0) / den * (b1 - b0);
  }
  return z;
}

// Importance resampling of the rays [first, first + count) of a warp's 32 rows, one
// warp-pass per ray.  (tnear, tfar, ray, valid) are this lane's own row's.  N = 2 slots per
// lane serve S <= 64, N = 4 (a separate kernel instantiation, so that its register needs
// do not touch the allocation of the common case's per-step loops) S <= 128.
struct ResampleArgs {
  const float* sc_w;
  float* sc_zf;
  float* z_fine;
  const float* noise_t;
  const float* noise_u;
  const float* frac;
  int S, wig;
  bool explicit_noise;
};
template <int N>
__device__ __forceinline__ void resample_rows_impl(const ResampleArgs& a, int first, int count,
                                                   float tnear, float tfar, size_t ray, bool valid,
                                                   int lane) {
  const int S = a.S;
  if (count <= 0) return;
  // inputs of ray j+1 are loaded while ray j is resampled
  struct In {
    LaneVec<N> w, n, u;
    size_t rayj;
  };
  auto load = [&](int j, In& in) {
    in.rayj = ((size_t)__shfl_sync(kFull, (unsigned)(ray >> 32), j) << 32) |
              (size_t)__shfl_sync(kFull, (unsigned)ray, j);
    const int col = 32 * a.wig + j;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const int e = 32 * i + lane;
      in.w.v[i] = (e < S) ? ldcg(a.sc_w + e * kThreads + col) : 0.f;
      in.n.v[i] = 0.f;
      if (a.explicit_noise) {
        in.n.v[i] = (e < S) ? a.noise_t[in.rayj * S + e] : 0.f;
        in.u.v[i] = (e < S) ? a.noise_u[in.rayj * S + e] : 2.f;
      } else {
        in.u.v[i] = (e < S) ? linspace01(e, S) : 2.f;
      }
    }
  };
  In cur, nxt;
  load(first, cur);
#pragma unroll 1
  for (int j = first; j < first + count; ++j) {
    load(j + 1 < first + count ? j + 1 : j, nxt);
    const float nearj = __shfl_sync(kFull, tnear, j), farj = __shfl_sync(kFull, tfar, j);
    const bool validj = __shfl_sync(kFull, (int)valid, j) != 0;
    const int col = 32 * a.wig + j;
    const float spanj = farj - nearj;
    LaneVec<N> t;
#pragma unroll
    for (int i = 0; i < N; ++i)
      t.v[i] = lerp_torch(nearj, farj, a.frac[32 * i + lane]) + cur.n.v[i] * (spanj / (float)S);
    const LaneVec<N> z = resample_ray<N>(cur.w, t, cur.u, !a.explicit_noise, S, lane);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const int e = 32 * i + lane;
      if (e < S) a.sc_zf[e * kThreads + col] = z.v[i];
      if (a.z_fine != nullptr && validj && e < S) a.z_fine[cur.rayj * S + e] = z.v[i];
    }
    cur = nxt;
  }
}
template <int NOUT_PAD, int EXTRA, bool FINE, int P, bool DBG, int NSLOT = 2, bool VD = false>
__global__ void __launch_bounds__(PipeCfg<P>::kThreadsTotal, 1)
render_forward_pipe(const nfi_render_params p, const unsigned char* __restrict__ wimg,
                    float* __restrict__ scratch) {
  using Cfg = PipeCfg<P, VD>;
  static_assert(!(VD && DBG), "the phase timers are not instantiated for the view-conditioned kernel");
  // VD: the image of nfi_layout.h; its `head` is what the shading group adds to a D2 row
  constexpr int kImgBytes = VD ? kVdBytes : kWiBytes;
  constexpr int kImgB1 = VD ? kVdB1 : kWiB1, kImgB2 = VD ? kVdHead : kWiB2;
  // extras composited with the weights: 3 world coordinates (EXTRA 1, recomputed from the
  // depth) or the NA attention probabilities (EXTRA 2, parked in scratch for the coarse samples)
  constexpr int NA_ = NOUT_PAD - 1;
  constexpr int NE = (EXTRA == 1) ? 3 : (EXTRA == 2 ? NA_ : 0);
  constexpr int NES = (EXTRA == 2) ? NA_ : 0;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* base = smem_raw;
  const int tid = threadIdx.x, lane = tid & 31;
  // Role by warpgroup.  The two consumer roles -- one warp each per sub-partition, nothing to
  // hide their latency behind -- sit above the producers: hardware wg 0..P-1 producer sets, P
  // shading, P+1 activation.  `wg` below is the logical role: 0 activation, 1 shading, 3..
  // producer sets (2 is unused).
  const int hw_wg = __shfl_sync(kFull, tid >> 7, 0);
  const int wg = (hw_wg < P) ? hw_wg + 3 : (P + 1 - hw_wg);
  const int gt = tid & 127;                        // row of the tile = ray
  const int wig = __shfl_sync(kFull, gt >> 5, 0);  // warp in warpgroup
  const int S = p.num_samples;

  uint64_t* bars = reinterpret_cast<uint64_t*>(base + Cfg::kSmBars);
  constexpr int NS = Cfg::kStages;
  uint64_t* full = bars;                         // [NS] stage gathered            (4 warps)
  uint64_t* a_free = full + NS;                  // [NS] stage loaded into registers (4 warps)
  uint64_t* d2_full = a_free + NS;               // [3]  D2 slot written           (4 warps)
  uint64_t* slot_free = d2_full + kPipeSlots;    // [3]  D2 read                   (4 warps)
  uint64_t* cw_ready = slot_free + kPipeSlots;   //      coarse weights of the tile written (4 warps)
  uint64_t* zf_ready = cw_ready + 1;             //      fine depths of the tile written (every resampling warp)
  uint64_t* wbar = zf_ready + 1;                 //      weight image landed
  float* d2s = reinterpret_cast<float*>(base + Cfg::kSmD2);  // [3][128][kD2Ld]
  const float* b1s = reinterpret_cast<const float*>(base + kImgB1);
  const float* b2s = reinterpret_cast<const float*>(base + kImgB2);
  float* pal = reinterpret_cast<float*>(base + Cfg::kSmPal);
  float* frac = reinterpret_cast<float*>(base + Cfg::kSmFrac);
  if (tid < 128) frac[tid] = (float)tid / (float)S;

  if (tid == 0) {
    if (tc::smem_u32(base) & 1023u) __trap();
    // barriers count WARPS: a warp-wide mbarrier.arrive is 32 serialised shared-memory atomics
    // on one word (L1 data-pipe wavefronts the gather needs)
    for (int i = 0; i < NS; ++i) {
      tc::mbar_init(&full[i], kWarps);
      tc::mbar_init(&a_free[i], kWarps);
    }
    for (int i = 0; i < kPipeSlots; ++i) {
      tc::mbar_init(&d2_full[i], kWarps);
      tc::mbar_init(&slot_free[i], kWarps);
    }
    tc::mbar_init(cw_ready, kWarps);
    tc::mbar_init(zf_ready, (2 + P) * kWarps);
    tc::mbar_init(wbar, 1);
    tc::fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    tc::mbar_expect_tx(wbar, kImgBytes);
    tc::tma_bulk_g2s(base, wimg, kImgBytes, wbar);
  }
  tc::mbar_wait(wbar, 0);

  const int tiles_x = (p.width + kTileW - 1) / kTileW;
  const int tiles_y = (p.height + kTileH - 1) / kTileH;
  const int n_tiles = tiles_x * tiles_y * p.batch;
  const int my_tiles =
      ((int)blockIdx.x < n_tiles) ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const uint32_t total_steps = (uint32_t)my_tiles * (uint32_t)S * (FINE ? 2u : 1u);
  const int R = p.plane_res;
  const float inv_range = 1.f / p.scene_range;
  const bool explicit_noise = (p.noise_mode == NFI_NOISE_EXPLICIT);
  // timing experiments only (bench.py --mlp-mode 0x104 / 0x204 / 0x804): results are garbage
  const bool dbg_skip_gather = (p.mlp_mode & 0x100) != 0;
  const bool dbg_skip_consumer = (p.mlp_mode & 0x200) != 0;
  const bool dbg_window = (p.mlp_mode & 0x800) != 0;
  // phase timers (DBG instantiation, mlp_mode & 0x1000, buffer in p.normals): lane 0 of
  // producer set 0 warp 0 -> [0..], activation warp 0 -> [16..], shading warp 0 -> [32..]
  const bool dbg_time = DBG && (p.mlp_mode & 0x1000) && p.normals != nullptr && blockIdx.x == 0 &&
                        lane == 0 && (wg <= 3) && wg != 2 && wig == 0;
  long long tacc[DBG ? 10 : 1];
  long long tprev = 0;
  if (DBG)
    for (int i = 0; i < 10; ++i) tacc[i] = 0;
#define NFI_T(i)                         \
  if (DBG && dbg_time) {                 \
    const long long now__ = clock64();   \
    tacc[i] += now__ - tprev;            \
    tprev = now__;                       \
  }
  float* slab = scratch + (size_t)blockIdx.x * pipe_scratch_floats(S, NES);
  float4* sc_srgb = reinterpret_cast<float4*>(slab);   // [S][128] coarse (sigma, r, g, b)
  float* sc_t = slab + (size_t)4 * S * kThreads;       // [S][128] coarse depths
  float* sc_w = sc_t + (size_t)S * kThreads;           // [S][128] coarse weights
  float* sc_zf = sc_w + (size_t)S * kThreads;          // [S][128] fine depths, ascending
  float* sc_e = sc_zf + (size_t)S * kThreads;          // [S][NES][128] coarse attention probabilities

  // Importance resampling of the rays [first, first + count) of this warp's 32 rows:
  // one warp-pass per ray.  (tnear, tfar, ray index, valid) are this lane's own row's.
  // The 32 rows of a quadrant are split over the 2 + P warps that serve it (shading,
  // activation and one warp of every producer set -- the producers would otherwise idle
  // between the coarse and the fine pass): a warp-pass is a chain of dependent shuffles at
  // ~0.1 IPC, so five warps per sub-partition get through the tile's 128 rays sooner than
  // two.
  constexpr int kRsParts = 2 + P;
  auto rs_first = [](int part) {  // part: 0 shading, 1 activation, 2.. producer sets
    constexpr int base_rows = 32 / kRsParts, rem = 32 % kRsParts;
    return part * base_rows + min(max(part - 2, 0), rem);
  };
  auto resample_rows = [&](int part, float tnear, float tfar, size_t ray, bool valid) {
    const int first = rs_first(part), count = rs_first(part + 1) - first;
    ResampleArgs ra;
    ra.sc_w = sc_w;
    ra.sc_zf = sc_zf;
    ra.z_fine = p.z_fine;
    ra.noise_t = p.noise_t;
    ra.noise_u = p.noise_u;
    ra.frac = frac;
    ra.S = S;
    ra.wig = wig;
    ra.explicit_noise = explicit_noise;
    resample_rows_impl<NSLOT>(ra, first, count, tnear, tfar, ray, valid, lane);
  };

  // The roles never share code after setmaxnreg: ptxas budgets registers per
  // region, and a block reachable from two branches gets the smaller count.
  if (wg >= 3) {
    // ================================ PRODUCER ================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::kProducerRegs));
    const int set = wg - 3;
    uint32_t n = 0;        // ring position at the start of the pass, identical in every role
    uint32_t tile_it = 0;  // tiles done by this CTA (parity of zf_ready)
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tile_it) {
      const TileCoord tcd = tile_coord(tile, tiles_x, tiles_y);
      const int b = tcd.b;
      int px, py;
      tile_pixel(tcd.tile_x, tcd.tile_y, wig, lane, px, py);
      const bool valid = (px < p.width) && (py < p.height);
      px = min(px, p.width - 1);
      py = min(py, p.height - 1);
      const size_t ray = ((size_t)b * p.height + py) * p.width + px;
      Ray r;
      setup_ray(p, b, py, px, r);
      const float span = r.tfar - r.tnear;
      const uint32_t plane_bytes = (uint32_t)R * (uint32_t)R * 128u;
      const unsigned char* planes_b =
          reinterpret_cast<const unsigned char*>(p.planes) + (size_t)b * 3 * plane_bytes;
      for (int pass = 0; pass < (FINE ? 2 : 1); ++pass) {
        if (pass == 1) {
          // this set's share of the quadrant's rows
          tc::mbar_wait(cw_ready, tile_it & 1);
          resample_rows(2 + set, r.tnear, r.tfar, ray, valid);
          __threadfence_block();
          __syncwarp();
          if (lane == 0) mbar_arrive(zf_ready);
          tc::mbar_wait(zf_ready, tile_it & 1);
        }
        // first step of this pass that belongs to this set; its sample value is
        // fetched one step ahead (the load is never waited on)
        int s = (int)(((uint32_t)set + (uint32_t)P - (n % P)) % P);
        auto fetch = [&](int ss) -> float {
          if (ss >= S) return 0.f;
          if (pass == 0) return explicit_noise ? p.noise_t[ray * S + ss] : 0.f;
          return ld_relaxed(sc_zf + ss * kThreads + gt);
        };
        float nxt = fetch(s);
        for (; s < S; s += P) {
          const uint32_t st = (n + (uint32_t)s) % NS, u = (n + (uint32_t)s) / NS;
          unsigned char* const stage = base + Cfg::kSmA + st * kFwdStageBytes;
          const float cur = nxt;
          nxt = fetch(s + P);
          if (DBG && dbg_time) tprev = clock64();
          NFI_STEP_WAIT(&a_free[st], (u & 1) ^ 1);  // tensor core has read the previous fill
          NFI_T(0)
          float t;
          if (pass == 0)
            t = lerp_torch(r.tnear, r.tfar, frac[s]) + cur * (span / (float)S);
          else
            t = cur;
          const float x0 = (r.ox + r.dx * t) * inv_range, x1 = (r.oy + r.dy * t) * inv_range,
                      x2 = (r.oz + r.dz * t) * inv_range;
          ByteTaps tp;
          byte_taps(x0, x1, R, 0u, tp.o[0], tp.fx[0], tp.fy[0]);
          byte_taps(x0, x2, R, plane_bytes >> 4, tp.o[1], tp.fx[1], tp.fy[1]);
          byte_taps(x1, x2, R, plane_bytes >> 3, tp.o[2], tp.fx[2], tp.fy[2]);
          NFI_T(1)
          if (dbg_window) {  // every tap inside a 32 KB window: L1 hits only
            tp.o[0] &= 0x7FFu;
            tp.o[1] &= 0x7FFu;
            tp.o[2] &= 0x7FFu;
          }
          if (!dbg_skip_gather)
            gather_to_tiles_lean<TileStore::kFp32>(planes_b, R, tp, stage, nullptr, 32 * wig, lane);
          NFI_T(2)
          // the stage is read with generic loads only (no async-proxy fence)
          __syncwarp();
          if (lane == 0) mbar_arrive(&full[st]);
          NFI_T(3)
          if (DBG && dbg_time) tacc[9] += 1;
        }
        n += (uint32_t)S;
      }
    }
    if (DBG && dbg_time)
      for (int i = 0; i < 10; ++i) p.normals[i] = (float)tacc[i];
  } else if (wg == 0) {
    // ================================ ACTIVATION ================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::kActRegs));
    const uint32_t base_s = tc::smem_u32(base);
    const uint64_t dsc_w1_hi = tc::gmma_desc_sw128(base_s + kWiW1Hi);
    const uint64_t dsc_w1_lo = tc::gmma_desc_sw128(base_s + kWiW1Lo);
    const uint64_t dsc_w2_hi = tc::gmma_desc_sw128(base_s + (VD ? kVdW2Hi : kWiW2Hi));
    const uint64_t dsc_w2_lo = tc::gmma_desc_sw128(base_s + (VD ? kVdW2Lo : kWiW2Lo));
    const float4* vt = reinterpret_cast<const float4*>(base + Cfg::kSmView) + gt;  // (VD only)
    uint32_t st = 0, u = 0, sl = 0, v = 0;
    // the next ring position: stage + D2 slot -> decoder -> d2_full, a_free
    auto activate = [&]() {
      if (DBG && dbg_time && tprev == 0) tprev = clock64();
      NFI_T(2)
      NFI_STEP_WAIT(&full[st], u & 1);
      NFI_STEP_WAIT(&slot_free[sl], (v & 1) ^ 1);
      NFI_T(0)
      float* d2 = d2s + sl * (kThreads * kD2Ld);
      if constexpr (VD) {
        decoder_step_vd(base + Cfg::kSmA + st * kFwdStageBytes, dsc_w1_hi, dsc_w1_lo, dsc_w2_hi,
                        dsc_w2_lo, tc::gmma_desc_sw128(base_s + kVdW3Hi),
                        tc::gmma_desc_sw128(base_s + kVdW3Lo), b1s, vt, d2, wig, lane, [&]() {
                          __syncwarp();
                          if (lane == 0) mbar_arrive(&a_free[st]);
                        });
      } else if (!dbg_skip_consumer) {
        decoder_step_fp32(base + Cfg::kSmA + st * kFwdStageBytes, dsc_w1_hi, dsc_w1_lo, dsc_w2_hi,
                          dsc_w2_lo, b1s, d2, wig, lane, [&]() {
                            __syncwarp();
                            if (lane == 0) mbar_arrive(&a_free[st]);
                          });
      } else {
        __syncwarp();
        if (lane == 0) mbar_arrive(&a_free[st]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&d2_full[sl]);
      if (++st == NS) { st = 0; ++u; }
      if (++sl == kPipeSlots) { sl = 0; ++v; }
      NFI_T(1)
      if (DBG && dbg_time) tacc[9] += 1;
    };
    uint32_t tile_it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tile_it) {
      if constexpr (VD)
        fill_view_tile(p, tile_coord(tile, tiles_x, tiles_y),
                       reinterpret_cast<const float*>(base + kVdB2f),
                       reinterpret_cast<float4*>(base + Cfg::kSmView) + gt, wig, lane);
      for (int s = 0; s < S; ++s) activate();
      if (FINE) {
        // second half of this warp's rows is resampled here, the first half by the
        // shading warp that owns them
        const TileCoord tcd = tile_coord(tile, tiles_x, tiles_y);
        int px, py;
        tile_pixel(tcd.tile_x, tcd.tile_y, wig, lane, px, py);
        const bool valid = (px < p.width) && (py < p.height);
        px = min(px, p.width - 1);
        py = min(py, p.height - 1);
        const size_t ray = ((size_t)tcd.b * p.height + py) * p.width + px;
        Ray r;
        setup_ray(p, tcd.b, py, px, r);
        tc::mbar_wait(cw_ready, tile_it & 1);
        NFI_T(3)
        resample_rows(1, r.tnear, r.tfar, ray, valid);
        __threadfence_block();
        __syncwarp();
        if (lane == 0) mbar_arrive(zf_ready);
        NFI_T(4)
        for (int s = 0; s < S; ++s) activate();
      }
    }
    if (DBG && dbg_time)
      for (int i = 0; i < 10; ++i) p.normals[16 + i] = (float)tacc[i];
  } else {
    // ================================ SHADING ================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::kShadeRegs));
    uint32_t sl = 0, v = 0;
    FieldConst fc;
    fc.A = p.n_attention;
    fc.use_sdf = p.use_sdf;
    fc.inv_beta = p.use_sdf ? 1.f / p.beta[0] : 0.f;
    fc.inv_alpha = p.use_sdf ? 1.f / p.alpha[0] : 0.f;

    uint32_t tile_it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tile_it) {
      const TileCoord tcd = tile_coord(tile, tiles_x, tiles_y);
      const int b = tcd.b;
      int px, py;
      tile_pixel(tcd.tile_x, tcd.tile_y, wig, lane, px, py);
      const bool valid = (px < p.width) && (py < p.height);
      px = min(px, p.width - 1);
      py = min(py, p.height - 1);
      const size_t ray = ((size_t)b * p.height + py) * p.width + px;
      Ray r;
      setup_ray(p, b, py, px, r);
      const float span = r.tfar - r.tnear;

      tc::bar_sync(1, kThreads);  // previous tile's palette no longer in use
      if (gt < 48)
        pal[gt] = (p.n_attention > 0 && gt < p.n_attention * 3)
                      ? p.palette[(size_t)b * p.n_attention * 3 + gt]
                      : 0.f;
      tc::bar_sync(1, kThreads);
      Compositor<NE, true> comp;
      comp.init();

      // decoder outputs of the next ring position -> density and colour at depth t
      auto shade = [&](float t, float& sigma, float& cr, float& cg, float& cb, float* ex) {
        const float* d2 = d2s + sl * (kThreads * kD2Ld) + gt * kD2Ld;
        if (DBG && dbg_time && tprev == 0) tprev = clock64();
        NFI_T(2)
        NFI_STEP_WAIT(&d2_full[sl], v & 1);
        NFI_T(0)
        float o16[16];
#pragma unroll
        for (int o4 = 0; o4 < 4; ++o4) {
          const float4 x = *reinterpret_cast<const float4*>(d2 + 4 * o4);
          o16[4 * o4] = x.x;
          o16[4 * o4 + 1] = x.y;
          o16[4 * o4 + 2] = x.z;
          o16[4 * o4 + 3] = x.w;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&slot_free[sl]);
        if (++sl == kPipeSlots) { sl = 0; ++v; }
        const float wx = r.ox + r.dx * t, wy = r.oy + r.dy * t, wz = r.oz + r.dz * t;
        const float x0 = wx * inv_range, x1 = wy * inv_range, x2 = wz * inv_range;
        const float keep =
            (fabsf(x0) > 1.f || fabsf(x1) > 1.f || fabsf(x2) > 1.f) ? 0.f : 1.f;
        float out[NOUT_PAD];
#pragma unroll
        for (int o4 = 0; o4 < NOUT_PAD / 4; ++o4) {
          const float4 bb = *reinterpret_cast<const float4*>(b2s + 4 * o4);
          out[4 * o4] = o16[4 * o4] + bb.x;
          out[4 * o4 + 1] = o16[4 * o4 + 1] + bb.y;
          out[4 * o4 + 2] = o16[4 * o4 + 2] + bb.z;
          out[4 * o4 + 3] = o16[4 * o4 + 3] + bb.w;
        }
        if (dbg_skip_consumer) {
          sigma = out[0];
          cr = cg = cb = out[1];
        } else {
          field_head_fast<NOUT_PAD>(out, fc, pal, keep, sigma, cr, cg, cb,
                                    EXTRA == 2 ? ex : nullptr);
        }
        if (EXTRA == 1) {
          ex[0] = wx;
          ex[1] = wy;
          ex[2] = wz;
        }
        NFI_T(1)
        if (DBG && dbg_time) tacc[9] += 1;
      };

      // ---------------- coarse pass ----------------
      {
        float wT = 1.f, prev_t = 0.f, prev_s = 0.f;
        // jitter: four steps per load, the next four in flight (S % 4 == 0)
        const float4* nz4 = reinterpret_cast<const float4*>(p.noise_t + ray * S);
        const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 nzc = explicit_noise ? nz4[0] : zero4;
        float4 nzn = (explicit_noise && S > 4) ? nz4[1] : zero4;
        const float jit = span / (float)S;
        for (int s = 0; s < S; ++s) {
          const int sq = s & 3;
          const float nz = sq == 0 ? nzc.x : (sq == 1 ? nzc.y : (sq == 2 ? nzc.z : nzc.w));
          const float t = lerp_torch(r.tnear, r.tfar, frac[s]) + nz * jit;
          if (sq == 3) {
            nzc = nzn;
            nzn = (explicit_noise && s + 5 < S) ? nz4[(s + 5) >> 2] : zero4;
          }
          float sigma, cr, cg, cb;
          float ex[NE > 0 ? NE : 1];
          shade(t, sigma, cr, cg, cb, ex);
          if (FINE) {
            sc_srgb[s * kThreads + gt] = make_float4(sigma, cr, cg, cb);
            sc_t[s * kThreads + gt] = t;
#pragma unroll
            for (int a = 0; a < NES; ++a) sc_e[((size_t)s * NES + a) * kThreads + gt] = ex[a];
            if (s > 0) {
              const float delta = (t - prev_t) * r.dn;
              const float a = 1.f - __expf(-prev_s * delta);
              sc_w[(s - 1) * kThreads + gt] = a * wT;
              wT = wT * ((1.f - a) + 1e-10f);
            }
            prev_t = t;
            prev_s = sigma;
          } else {
            comp.push(t, sigma, cr, cg, cb, ex, r.dn);
          }
          NFI_T(3)
        }
      }

      if (FINE) {
        sc_w[(S - 1) * kThreads + gt] = 0.f;
        __threadfence_block();
        __syncwarp();
        if (lane == 0) mbar_arrive(cw_ready);  // the activation group may resample its half
        tc::mbar_wait(cw_ready, tile_it & 1);
        NFI_T(4)
        resample_rows(0, r.tnear, r.tfar, ray, valid);
        __threadfence_block();
        __syncwarp();
        if (lane == 0) mbar_arrive(zf_ready);  // (with the activation group's 4) producers may start
        tc::mbar_wait(zf_ready, tile_it & 1);
        NFI_T(5)

        // ------- fine pass + sorted merge + compositing -------
        // The next TWO coarse samples wait in registers, so taking one never
        // stalls on the (L2) load of its successor.
        int c = 0;
        float ct0 = ldcg(sc_t + gt), ct1 = ldcg(sc_t + kThreads + gt);
        float4 cq0 = __ldcg(sc_srgb + gt), cq1 = __ldcg(sc_srgb + kThreads + gt);
        auto take_coarse = [&]() {
          float ce[NE > 0 ? NE : 1];
          if (EXTRA == 1) {
            ce[0] = r.ox + r.dx * ct0;
            ce[1] = r.oy + r.dy * ct0;
            ce[2] = r.oz + r.dz * ct0;
          }
#pragma unroll
          for (int a = 0; a < NES; ++a) ce[a] = ldcg(sc_e + ((size_t)c * NES + a) * kThreads + gt);
          comp.push(ct0, cq0.x, cq0.y, cq0.z, cq0.w, ce, r.dn);
          ++c;
          ct0 = ct1;
          cq0 = cq1;
          if (c + 1 < S) {
            ct1 = ldcg(sc_t + (c + 1) * kThreads + gt);
            cq1 = __ldcg(sc_srgb + (c + 1) * kThreads + gt);
          }
        };
        float z0 = ldcg(sc_zf + gt);
        float z1 = (S > 1) ? ldcg(sc_zf + kThreads + gt) : 0.f;
        for (int k = 0; k < S; ++k) {
          const float z = z0;
          z0 = z1;
          z1 = (k + 2 < S) ? ldcg(sc_zf + (k + 2) * kThreads + gt) : 0.f;
          float sigma, cr, cg, cb;
          float ex[NE > 0 ? NE : 1];
          shade(z, sigma, cr, cg, cb, ex);
          while (c < S && ct0 <= z) take_coarse();
          comp.push(z, sigma, cr, cg, cb, ex, r.dn);
          NFI_T(3)
        }
        while (c < S) take_coarse();
        NFI_T(6)
      }

      if (valid) {
        float bg = 0.f;
        if (p.white_background) bg = 1.f - comp.am;
        p.rgb[ray * 3 + 0] = comp.ar + bg;
        p.rgb[ray * 3 + 1] = comp.ag + bg;
        p.rgb[ray * 3 + 2] = comp.ab + bg;
        p.depth[ray] = comp.ad;
        p.mask[ray] = comp.am;
        // the exchange step of the multi-GPU form, fused: the same five floats go to this ray's
        // place in every peer's full-batch buffers over NVLink (posted stores; the ranks meet at
        // a barrier after the kernel, parallel.PeerExchange)
        for (int q = 0; q < p.n_peers; ++q) {
          float* pr = p.peer_rgb[q] + ray * 3;
          pr[0] = comp.ar + bg;
          pr[1] = comp.ag + bg;
          pr[2] = comp.ab + bg;
          p.peer_depth[q][ray] = comp.ad;
          p.peer_mask[q][ray] = comp.am;
        }
        if (EXTRA == 1 && p.extra != nullptr)
          for (int a = 0; a < 3; ++a) p.extra[ray * 3 + a] = comp.ae[a];
        if (EXTRA == 2 && p.extra != nullptr)
          for (int a = 0; a < NE; ++a)
            if (a < p.n_attention) p.extra[ray * p.n_attention + a] = comp.ae[a];
      }
    }
    if (DBG && dbg_time)
      for (int i = 0; i < 10; ++i) p.normals[32 + i] = (float)tacc[i];
  }
#undef NFI_T
  __syncthreads();
  if (p.n_peers > 0 && p.peer_done != nullptr && tid == 0) {
    // Completion handshake of the fused exchange.  Every CTA: its threads' peer stores are ordered
    // before the bar.sync above, the system-scope fence publishes them, then it counts itself.
    // The last CTA of this rank signals every peer and waits for their signals: a completed
    // kernel means "all ranks' tiles have landed here".
    __threadfence_system();
    const unsigned done = atomicAdd(p.peer_done, 1u);
    if (done == gridDim.x - 1) {
      __threadfence();
      *p.peer_done = 0u;
      for (int q = 0; q < p.n_peers; ++q)
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p.peer_signal[q]), "r"(p.peer_epoch)
                     : "memory");
      const long long t0 = clock64();
      for (int q = 0; q < p.n_peers; ++q) {
        const uint32_t* flag = p.peer_signal_self + p.peer_rank[q];
        uint32_t v;
        do {
          asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
          if ((int)(v - p.peer_epoch) >= 0) break;
          __nanosleep(200);
          if (clock64() - t0 > 60000000000LL) __trap();  // (~30 s) a peer never arrived: fail, do not hang
        } while (true);
      }
    }
  }
}

}  // namespace nfi
