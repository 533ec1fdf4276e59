// Decoder-weight gradients on the tensor cores (SURVEY.md section 8 row a13; the GAN generator
// step, run.py:1044: loss.backward() with the decoder trainable).
//
//   dW1[j][c] = sum_points dpre[p][j] F[p][c]      db1[j] = sum_points dpre[p][j]
//   dW2[o][j] = sum_points dOut[p][o] H[p][j]      db2[o] = sum_points dOut[p][o]
//
// are contractions over the POINTS, i.e. over what the other GEMMs of the path keep as the M
// dimension.  wgmma reads MN-major ("transposed") operands from shared memory for 16-bit types,
// so every operand of a step is laid down point-major as a bf16 hi/lo PAIR (2^-17: these sums are
// dominated by a few very large terms; single bf16 operands leave 1e-3, pairs 3e-5 against the
// fp32 kernel) and five accumulating wgmma per 16 points and 64 rows form
//
//   XA = [ dpre_hi (64) | dpre_lo (64) ]   XB = [ H_hi (64) | H_lo (64) ]      (A operands)
//   += XA^T F_hi,  += XA^T F_lo      rows j and 64 + j together: dW1[j][.]
//   += XB^T dOut_hi, += XB^T dOut_lo   rows j and 64 + j together: dW2[.][j]
//   += XA^T 1                          db1[j]
//
// in the registers of a warpgroup of their own (56 accumulators per thread), cut into chains of
// kWgFlush steps that are banked in fp32 (below) and added to the global gradients once per CTA.
// db2 is summed in fp32 registers by the shading threads.
//
// To make room for the pair tiles, layer 1 of the recompute chain runs on bf16 pairs too (as the
// synthesis convolutions do): the gather writes the features as two [128][32 bf16] SWIZZLE_64B
// tiles (16 KB per stage instead of 32) that are BOTH the K-major A operand of MMA1 and, rows = K,
// the MN-major B operand of the dW1 products.  The rest of the chain is render_backward_pipe's
// (MMA2 / MMA3 / MMA4 in 3xTF32 with register A fragments, softplus and its reverse, reverse
// compositing, issued by the activation warpgroup).  Two forms:
//   PLANES = true  (the generator step: decoder AND planes / palette / beta / alpha gradients,
//                   cameras are data): MMA4 and the scatter of render_backward_pipe are folded
//                   in -- ONE sweep;
//   PLANES = false (decoder gradients only, or a pose gradient is wanted too): this kernel beside
//                   render_backward_pipe, which then sees the decoder as a constant.
// The accumulator warpgroup costs the register file what a second producer set would need, so
// one producer set serves the sweep.
#pragma once
#include <cuda_bf16.h>

#include "nfi_backward_pipe.cuh"

namespace nfi {

constexpr int kWgSlots = 2;
constexpr int kWgStages = 3;
// The tensor core adds into its accumulator with truncation, a bias that grows with the length
// of the chain; a CTA of config 2 would chain 28,000 accumulating MMAs = 450,000 terms.  The
// chain is therefore cut every kWgFlush steps (2,048 terms): the accumulator is added, in fp32
// round-to-nearest, to a per-CTA row buffer in global memory (L2-resident, single writer per
// element) and the next chain starts from zero.
constexpr int kWgFlush = 16;
constexpr size_t kWgAccBytesPerCta = 128 * 64 * sizeof(float);

// PLANES: the kernel also forms dL/d(texel features) (MMA4) and scatters it into the plane
// gradient, and accumulates the palette / beta / alpha gradients -- i.e. it is the WHOLE backward
// of the GAN generator step in one sweep (no pose gradient: cameras are data there).
template <bool PLANES>
struct WgCfgT {
  static constexpr int P = 1;
  static constexpr int kThreadsTotal = 384 + 128 * P;  // producers, accumulators, shading, activation
  static constexpr int kStageBytes = 16384;                           // F_hi | F_lo, 8 KB each
  static constexpr int kWbBytes = PLANES ? 32768 : 16384;             // W2^T hi/lo (+ W1^T/3 hi/lo)
  static constexpr int kSmWb = 25600;
  static constexpr int kSmW1 = kSmWb + kWbBytes;                      // W1 bf16 hi | lo (8 KB)
  static constexpr int kSmA = kSmW1 + 8192;
  static constexpr int kSmX = kSmA + kWgStages * kStageBytes;         // 4 x 16 KB
  static constexpr int kSmE = kSmX + 65536;                           // dOut hi | lo
  static constexpr int kSmOnes = kSmE + 8192;                         // 1 KB of 1.0
  static constexpr int kSmD2 = kSmOnes + 1024;                        // D2 / dOut slots
  static constexpr int kSmD4 = kSmD2 + kWgSlots * kD2SlotBytes;       // one D4 slot (PLANES)
  static constexpr int kSmPal = kSmD4 + (PLANES ? kD4SlotBytes : 0);
  static constexpr int kSmFrac = kSmPal + 48 * 4;
  static constexpr int kSmBars = kSmFrac + 128 * 4;
  // full[3], a_free[3], per slot: d2_full, dout_ready; d4_full, d4_free; x_ready, x_free;
  // weights x2
  static constexpr int kNumBars = 2 * kWgStages + 2 * kWgSlots + 2 + 2 + 2;
  static constexpr int kSmBytes = kSmBars + kNumBars * 8;
  // 512 x 128 = 65536 = 128 x (112 + 120 + 136 + 144) = 128 x (96 + 120 + 136 + 160)
  static constexpr int kProdRegs = PLANES ? 112 : 96;
  static constexpr int kAccRegs = 120;
  static constexpr int kShadeRegs = 136;
  static constexpr int kActRegs = PLANES ? 144 : 160;
};
using WgCfg = WgCfgT<false>;
static_assert(WgCfgT<true>::kSmBytes <= 227 * 1024, "shared memory budget");
static_assert((WgCfgT<false>::kSmA & 1023) == 0 && (WgCfgT<false>::kSmX & 1023) == 0 &&
                  (WgCfgT<false>::kSmE & 1023) == 0 && (WgCfgT<false>::kSmW1 & 1023) == 0 &&
                  (WgCfgT<true>::kSmA & 1023) == 0 && (WgCfgT<true>::kSmX & 1023) == 0 &&
                  (WgCfgT<true>::kSmE & 1023) == 0 && (WgCfgT<true>::kSmW1 & 1023) == 0,
              "swizzled tiles are 1024-byte aligned");


template <int NOUT_PAD, bool PLANES = false>
__global__ void __launch_bounds__(WgCfgT<PLANES>::kThreadsTotal, 1)
render_wgrad_pipe(const nfi_render_params p, const nfi_render_grads g,
                  const unsigned char* __restrict__ wimg, float* __restrict__ acc_ws) {
  using Cfg = WgCfgT<PLANES>;
  constexpr int P = Cfg::P;
  constexpr int NA = NOUT_PAD - 1;
  constexpr int NS = kWgStages;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* base = smem_raw;
  const int tid = threadIdx.x, lane = tid & 31;
  const int hw_wg = __shfl_sync(kFull, tid >> 7, 0);
  // logical role: 0 activation, 1 shading, 2 weight-gradient accumulators, 3.. producer sets
  const int wg = (hw_wg < P) ? hw_wg + 3 : (P + 2 - hw_wg);
  const int gt = tid & 127;
  const int wig = __shfl_sync(kFull, gt >> 5, 0);
  const int S = p.num_samples;
  const int n_total = (p.fine_sampling ? 2 : 1) * S;  // steps per tile

  uint64_t* bars = reinterpret_cast<uint64_t*>(base + Cfg::kSmBars);
  uint64_t* full = bars;                      // [3] stage gathered (4 warps)
  uint64_t* a_free = full + NS;               // [3] stage read by the activation AND dW GEMMs (8 warps)
  uint64_t* d2_full = a_free + NS;            // [2] D2 in its slot (4 warps)
  uint64_t* dout_ready = d2_full + kWgSlots;  // [2] dOut in the slot and in the E tiles (4 warps)
  uint64_t* d4_full = dout_ready + kWgSlots;  //     D4 in its slot (PLANES, 4 warps)
  uint64_t* d4_free = d4_full + 1;            //     D4 scattered (PLANES, 4 warps)
  uint64_t* x_ready = d4_free + 1;            //     X tiles written (4 warps)
  uint64_t* x_free = x_ready + 1;             //     X and E tiles read by the dW GEMMs (4 warps)
  uint64_t* wbar = x_free + 1;                // [2] weight images landed
  float* d2s = reinterpret_cast<float*>(base + Cfg::kSmD2);  // [2][128][kD2Ld]
  float* d4s = reinterpret_cast<float*>(base + Cfg::kSmD4);  // [128][kD4Ld]
  const float* b1s = reinterpret_cast<const float*>(base + kWiB1);
  const float* b2s = reinterpret_cast<const float*>(base + kWiB2);
  float* pal = reinterpret_cast<float*>(base + Cfg::kSmPal);
  float* frac = reinterpret_cast<float*>(base + Cfg::kSmFrac);
  if (tid < 128) frac[tid] = (float)tid / (float)S;
  // constants in shared memory: 1 KB of bf16 ones (the B operand of db1) and layer 1's weights
  // (x log2 e, as the forward weight image has them) as a bf16 hi / lo pair, [64 rows = hidden
  // unit][32 k] K-major SWIZZLE_64B
  for (int i = tid; i < 256; i += Cfg::kThreadsTotal)
    reinterpret_cast<uint32_t*>(base + Cfg::kSmOnes)[i] = 0x3F803F80u;
  for (int i = tid; i < kHid * kC; i += Cfg::kThreadsTotal) {
    const int j = i / kC, c = i % kC;
    const float w = p.w1[i] * kLog2e;
    const __nv_bfloat16 hi = __float2bfloat16_rn(w);
    const __nv_bfloat16 lo = __float2bfloat16_rn(w - __bfloat162float(hi));
    const uint32_t off = tc::sw64_offset(j, c >> 3) + (c & 7) * 2;
    *reinterpret_cast<__nv_bfloat16*>(base + Cfg::kSmW1 + off) = hi;
    *reinterpret_cast<__nv_bfloat16*>(base + Cfg::kSmW1 + 4096 + off) = lo;
  }
  tc::fence_async_smem();
  if (tid == 0) {
    if (tc::smem_u32(base) & 1023u) __trap();
    for (int i = 0; i < NS; ++i) {
      tc::mbar_init(&full[i], kWarps);
      tc::mbar_init(&a_free[i], 2 * kWarps);
    }
    for (int i = 0; i < kWgSlots; ++i) {
      tc::mbar_init(&d2_full[i], kWarps);
      tc::mbar_init(&dout_ready[i], kWarps);
    }
    tc::mbar_init(d4_full, kWarps);
    tc::mbar_init(d4_free, kWarps);
    tc::mbar_init(x_ready, kWarps);
    tc::mbar_init(x_free, kWarps);
    tc::mbar_init(&wbar[0], 1);
    tc::mbar_init(&wbar[1], 1);
    tc::fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    tc::mbar_expect_tx(&wbar[0], kWiBytes);
    tc::tma_bulk_g2s(base, wimg, kWiBytes, &wbar[0]);
    tc::mbar_expect_tx(&wbar[1], Cfg::kWbBytes);
    tc::tma_bulk_g2s(base + Cfg::kSmWb, wimg + 32768, Cfg::kWbBytes, &wbar[1]);  // W2^T (| W1^T / 3)
  }
  tc::mbar_wait(&wbar[0], 0);
  tc::mbar_wait(&wbar[1], 0);

  const int tiles_x = (p.width + kTileW - 1) / kTileW;
  const int tiles_y = (p.height + kTileH - 1) / kTileH;
  const int n_tiles = tiles_x * tiles_y * p.batch;
  const int my_tiles =
      ((int)blockIdx.x < n_tiles) ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const uint32_t total_steps = (uint32_t)my_tiles * (uint32_t)n_total;
  const int R = p.plane_res;
  const float inv_range = 1.f / p.scene_range;
  const uint32_t plane_bytes = (uint32_t)R * (uint32_t)R * 128u;

  if (wg >= 3) {
    // ================================ PRODUCERS (gather; PLANES: also the scatter) ================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::kProdRegs));
    const int set = wg - 3;
    const int q = lane >> 3, kq = lane & 7;
    const uint32_t row_units = (uint32_t)R * 8u;
    uint32_t n0 = 0;  // ring position of the tile's first step
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, n0 += (uint32_t)n_total) {
      const TileCoord tcd = tile_coord(tile, tiles_x, tiles_y);
      const int b = tcd.b;
      int px, py;
      tile_pixel(tcd.tile_x, tcd.tile_y, wig, lane, px, py);
      px = min(px, p.width - 1);
      py = min(py, p.height - 1);
      const size_t ray = ((size_t)b * p.height + py) * p.width + px;
      Ray r;
      setup_ray(p, b, py, px, r);
      const unsigned char* planes_b =
          reinterpret_cast<const unsigned char*>(p.planes) + (size_t)b * 3 * plane_bytes;
      float* gplanes_b = (PLANES && g.grad_planes)
                             ? g.grad_planes + (size_t)b * 3 * (plane_bytes >> 2) : nullptr;
      MergeWalk mw;
      mw.init(p, r, ray, frac);
      int walked = 0;
      ByteTaps cur, nxt;  // taps of the (up to) two steps this set has between "gathered" and "scattered"
      auto gather_step = [&](int i, ByteTaps& tp) {
        float z = 0.f;
        while (walked <= i) {
          z = mw.pop();
          ++walked;
        }
        const float x0 = (r.ox + r.dx * z) * inv_range, x1 = (r.oy + r.dy * z) * inv_range,
                    x2 = (r.oz + r.dz * z) * inv_range;
        byte_taps(x0, x1, R, 0u, tp.o[0], tp.fx[0], tp.fy[0]);
        byte_taps(x0, x2, R, plane_bytes >> 4, tp.o[1], tp.fx[1], tp.fy[1]);
        byte_taps(x1, x2, R, plane_bytes >> 3, tp.o[2], tp.fx[2], tp.fy[2]);
        const uint32_t m = n0 + (uint32_t)i;
        const uint32_t st = m % NS, u = m / NS;
        unsigned char* const stage = base + Cfg::kSmA + st * Cfg::kStageBytes;
        NFI_STEP_WAIT(&a_free[st], (u & 1) ^ 1);
        gather_to_tiles_lean<true>(planes_b, R, tp, stage, stage + 8192, 32 * wig, lane);
        tc::fence_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&full[st]);
      };
      if constexpr (!PLANES) {
        for (int i = set; i < n_total; i += P) gather_step(i, cur);
      } else {
        if (set < n_total) gather_step(set, cur);
        for (int i = set; i < n_total; i += P) {
          if (i + P < n_total) gather_step(i + P, nxt);
          // ---- scatter step i: D4 -> plane gradient (as render_backward_pipe, no pose gradient)
          const uint32_t m = n0 + (uint32_t)i;
          // this warp's 32 rows of the D4 slot, read in place (released after the scatter)
          const float* Dw = d4s + 32 * wig * kD4Ld;
          NFI_STEP_WAIT(d4_full, m & 1);
          if (gplanes_b != nullptr) {
#pragma unroll 1
            for (int gq = 0; gq < 8; ++gq) {
              const int src = 4 * gq + q;
              const float4 d4v = *reinterpret_cast<const float4*>(Dw + src * kD4Ld + 4 * kq);
#pragma unroll
              for (int pl = 0; pl < 3; ++pl) {
                const uint32_t a00 = __shfl_sync(kFull, cur.o[pl], src) | (uint32_t)kq;
                const float fx = __shfl_sync(kFull, cur.fx[pl], src);
                const float fy = __shfl_sync(kFull, cur.fy[pl], src);
                const float gx0 = 1.f - fx, gy0 = 1.f - fy;
                const float w00 = gx0 * gy0, w01 = fx * gy0, w10 = gx0 * fy, w11 = fx * fy;
                float* gp = gplanes_b;
                red_add_v4(gp + (size_t)a00 * 4, d4v.x * w00, d4v.y * w00, d4v.z * w00, d4v.w * w00);
                red_add_v4(gp + (size_t)(a00 + 8u) * 4, d4v.x * w01, d4v.y * w01, d4v.z * w01,
                           d4v.w * w01);
                red_add_v4(gp + (size_t)(a00 + row_units) * 4, d4v.x * w10, d4v.y * w10,
                           d4v.z * w10, d4v.w * w10);
                red_add_v4(gp + (size_t)(a00 + row_units + 8u) * 4, d4v.x * w11, d4v.y * w11,
                           d4v.z * w11, d4v.w * w11);
              }
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(d4_free);
          cur = nxt;
        }
      }
    }
  } else if (wg == 2) {
    // ================================ WEIGHT-GRADIENT ACCUMULATORS ================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::kAccRegs));
    const uint32_t base_s = tc::smem_u32(base);
    const int g4 = lane >> 2, t = lane & 3;
    // accumulator row r = 64 mb + 16 wig + g4 (+ 8) = hidden unit j (mb 0: dpre_hi / H_hi rows, 1:
    // the lo halves): dW1[j][c] at columns c, dW2[o][j] at o, db1[j] (all 8 columns equal)
    float w1a[2][16], w2a[2][8], b1a[2][4];
    auto clear = [&]() {
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) {
        zero(w1a[mb]);
        zero(w2a[mb]);
        zero(b1a[mb]);
      }
    };
    // the row buffer of this CTA ([128][64]: columns 0..31 dW1, 32..47 dW2, 48 db1): `first`: it
    // is written, not added to; `final`: the total goes to the global gradients instead
    const int nout_w = 1 + (p.n_attention > 0 ? p.n_attention : 3);
    auto flush = [&](bool first, bool final) {
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int row = 64 * mb + 16 * wig + g4 + 8 * half, j = row & (kHid - 1);
          float* const myrow = acc_ws + ((size_t)blockIdx.x * 128 + row) * 64;
          auto put = [&](int col, float a, float b, float* gdst0, float* gdst1) {
            float2 v2 = make_float2(a, b);
            if (!first) {
              const float2 o = *reinterpret_cast<const float2*>(myrow + col);
              v2.x += o.x;
              v2.y += o.y;
            }
            if (!final) {
              *reinterpret_cast<float2*>(myrow + col) = v2;
            } else {
              if (gdst0) atomicAdd(gdst0, v2.x);
              if (gdst1) atomicAdd(gdst1, v2.y);
            }
          };
#pragma unroll
          for (int jb = 0; jb < 4; ++jb) {
            const int c = 8 * jb + 2 * t;
            put(c, w1a[mb][4 * jb + 2 * half], w1a[mb][4 * jb + 2 * half + 1],
                g.grad_w1 ? g.grad_w1 + j * kC + c : nullptr,
                g.grad_w1 ? g.grad_w1 + j * kC + c + 1 : nullptr);
          }
#pragma unroll
          for (int jb = 0; jb < 2; ++jb) {
            const int o = 8 * jb + 2 * t;
            put(32 + o, w2a[mb][4 * jb + 2 * half], w2a[mb][4 * jb + 2 * half + 1],
                (g.grad_w2 && o < nout_w) ? g.grad_w2 + o * kHid + j : nullptr,
                (g.grad_w2 && o + 1 < nout_w) ? g.grad_w2 + (o + 1) * kHid + j : nullptr);
          }
          if (t == 0) put(48, b1a[mb][2 * half], 0.f, g.grad_b1 ? g.grad_b1 + j : nullptr, nullptr);
        }
      }
    };
    clear();
    const uint64_t dsc_one = tc::gmma_desc(base_s + Cfg::kSmOnes, tc::kSw32, 16, 256);
    uint32_t st = 0, u = 0, sl = 0, v = 0;
    for (uint32_t m = 0; m < total_steps; ++m) {
      NFI_STEP_WAIT(&full[st], u & 1);
      NFI_STEP_WAIT(&dout_ready[sl], v & 1);
      NFI_STEP_WAIT(x_ready, m & 1);
      const uint32_t stage_s = base_s + Cfg::kSmA + st * Cfg::kStageBytes;
      tc::wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {  // 16 points: 2048 B of X, 1024 B of F, 512 B of dOut
        // MN-major operands: rows = points (K)
        const uint64_t f_hi = tc::gmma_desc(stage_s + 1024 * ks, tc::kSw64, 16, 512);
        const uint64_t f_lo = tc::gmma_desc(stage_s + 8192 + 1024 * ks, tc::kSw64, 16, 512);
        const uint64_t e_hi = tc::gmma_desc(base_s + Cfg::kSmE + 512 * ks, tc::kSw32, 16, 256);
        const uint64_t e_lo = tc::gmma_desc(base_s + Cfg::kSmE + 4096 + 512 * ks, tc::kSw32, 16, 256);
#pragma unroll
        for (int mb = 0; mb < 2; ++mb) {
          const uint32_t xa_s = base_s + Cfg::kSmX + 16384 * mb + 2048 * ks;
          const uint64_t xa = tc::gmma_desc(xa_s, tc::kSw128, 16, 1024);
          const uint64_t xb = tc::gmma_desc(xa_s + 32768, tc::kSw128, 16, 1024);
          tc::wgmma_bf16_ss_n32<1, 1>(w1a[mb], xa, f_hi, 1);
          tc::wgmma_bf16_ss_n32<1, 1>(w1a[mb], xa, f_lo, 1);
          tc::wgmma_bf16_ss_n8<1, 0>(b1a[mb], xa, dsc_one, 1);
          tc::wgmma_bf16_ss_n16<1, 1>(w2a[mb], xb, e_hi, 1);
          tc::wgmma_bf16_ss_n16<1, 1>(w2a[mb], xb, e_lo, 1);
        }
      }
      tc::wgmma_commit();
      tc::wgmma_wait<0>();
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) {
        tc::reg_fence(w1a[mb]);
        tc::reg_fence(w2a[mb]);
        tc::reg_fence(b1a[mb]);
      }
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&a_free[st]);
        mbar_arrive(x_free);
      }
      if ((m + 1) % kWgFlush == 0 && m + 1 < total_steps) {
        flush(m + 1 == (uint32_t)kWgFlush, false);
        clear();
      }
      if (++st == NS) { st = 0; ++u; }
      if (++sl == kWgSlots) { sl = 0; ++v; }
    }
    // ---- the last chain + the banked ones -> global gradients (one atomic per entry per CTA)
    if (total_steps > 0) flush(total_steps <= (uint32_t)kWgFlush, true);
  } else if (wg == 0) {
    // ================================ ACTIVATION (forward and reverse) ================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::kActRegs));
    unsigned char* const xrow = base + Cfg::kSmX;
    const uint32_t base_s = tc::smem_u32(base);
    const uint64_t w1_hi = tc::gmma_desc(base_s + Cfg::kSmW1, tc::kSw64, 16, 512);
    const uint64_t w1_lo = tc::gmma_desc(base_s + Cfg::kSmW1 + 4096, tc::kSw64, 16, 512);
    const uint64_t w2_hi = tc::gmma_desc_sw128(base_s + kWiW2Hi);
    const uint64_t w2_lo = tc::gmma_desc_sw128(base_s + kWiW2Lo);
    const uint64_t b3_hi = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kWbW2tHi);
    const uint64_t b3_lo = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kWbW2tLo);
    const uint64_t b4_hi = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kWbW1tHi);
    const uint64_t b4_lo = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kWbW1tLo);
    const int g4 = lane >> 2, t = lane & 3;
    // layer 1 on bf16 pairs for the 64 rows of block mb: D1 = F_lo W1_hi + F_hi W1_lo + F_hi W1_hi,
    // K = 32 = two K16 steps of 32 bytes
    auto layer1 = [&](float (&d)[32], uint32_t stage_s, int mb) {
      const uint64_t a_hi = tc::gmma_desc(stage_s + 4096 * mb, tc::kSw64, 16, 512);
      const uint64_t a_lo = tc::gmma_desc(stage_s + 8192 + 4096 * mb, tc::kSw64, 16, 512);
      tc::wgmma_bf16_ss_n64<0, 0>(d, a_lo, w1_hi, 0);
      tc::wgmma_bf16_ss_n64<0, 0>(d, a_lo + 2, w1_hi + 2, 1);
      tc::wgmma_bf16_ss_n64<0, 0>(d, a_hi, w1_lo, 1);
      tc::wgmma_bf16_ss_n64<0, 0>(d, a_hi + 2, w1_lo + 2, 1);
      tc::wgmma_bf16_ss_n64<0, 0>(d, a_hi, w1_hi, 1);
      tc::wgmma_bf16_ss_n64<0, 0>(d, a_hi + 2, w1_hi + 2, 1);
    };
    auto act_fwd = [&](uint32_t m) {
      const uint32_t st = m % NS, u = m / NS, sl = m % kWgSlots;
      const uint32_t stage_s = base_s + Cfg::kSmA + st * Cfg::kStageBytes;
      float* d2 = d2s + sl * (kThreads * kD2Ld);
      NFI_STEP_WAIT(&full[st], u & 1);
#pragma unroll 1
      for (int mb = 0; mb < 2; ++mb) {
        float d[32];
        zero(d);
        tc::wgmma_fence();
        layer1(d, stage_s, mb);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::reg_fence(d);
        uint32_t hi[8][4], lo[8][4];
        tc::softplus_frag<true>(d, b1s, t, hi, lo);
        float o[8];
        zero(o);
        tc::wgmma_fence();
        tc::layer2_mb(o, hi, lo, w2_hi, w2_lo);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::reg_fence(o);
        tc::store_frag_rows(o, d2 + 64 * mb * kD2Ld, kD2Ld, wig, lane);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&d2_full[sl]);
    };
    // dpre = dH * sigmoid(pre),  sigmoid(pre) = 1 - exp(-softplus(pre)); dpre and H go to the
    // X tiles as bf16 hi / lo pairs (row = point, MN-major atoms of 64 columns); PLANES: D4 too
    auto act_bwd = [&](uint32_t m) {
      const uint32_t st = m % NS, sl = m % kWgSlots, v = m / kWgSlots;
      const uint32_t stage_s = base_s + Cfg::kSmA + st * Cfg::kStageBytes;
      const float* dout = d2s + sl * (kThreads * kD2Ld);
      NFI_STEP_WAIT(&dout_ready[sl], v & 1);
      NFI_STEP_WAIT(x_free, (m & 1) ^ 1);  // the previous step's dW GEMMs have read the X tiles
      if constexpr (PLANES) NFI_STEP_WAIT(d4_free, (m & 1) ^ 1);  // D4 of step m - 1 scattered
#pragma unroll 1
      for (int mb = 0; mb < 2; ++mb) {
        float d[32], d3[32];
        zero(d);
        zero(d3);
        uint32_t ohi[2][4], olo[2][4];
        load_dout_frags(dout + 64 * mb * kD2Ld, wig, lane, ohi, olo);
        tc::wgmma_fence();
        layer1(d, stage_s, mb);
        mma3_mb(d3, ohi, olo, b3_hi, b3_lo);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::reg_fence(d);
        tc::reg_fence(d3);
        if (mb == 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&a_free[st]);
        }
        uint32_t phi[8][4], plo[8][4];
#pragma unroll
        for (int kb = 0; kb < 8; ++kb) {
          const float2 bb = *reinterpret_cast<const float2*>(b1s + 8 * kb + 2 * t);
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            float hv[2], dp[2];
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int e = 2 * half + c;
              hv[c] = tc::softplus_mufu<true>(d[4 * kb + e] + (c ? bb.y : bb.x));
              const float sg = 1.f - tc::ex2_approx(-hv[c] * kLog2e);
              dp[c] = d3[4 * kb + e] * sg;
              if constexpr (PLANES) tc::put_split(phi, plo, kb, tc::afrag_slot(e), dp[c]);
            }
            // columns 8kb + 2t, +1 of this thread's row in dpre_hi / dpre_lo (tiles 0, 1) and
            // H_hi / H_lo (tiles 2, 3)
            const int row = 64 * mb + 16 * wig + g4 + 8 * half;
            const uint32_t off = tc::sw128_offset(row, kb) + 4 * t;
            const uint32_t dh = tc::bf16x2_rn(dp[0], dp[1]);
            const uint32_t dl = tc::bf16x2_rn(dp[0] - __uint_as_float(dh << 16),
                                              dp[1] - __uint_as_float(dh & 0xFFFF0000u));
            const uint32_t hh = tc::bf16x2_rn(hv[0], hv[1]);
            const uint32_t hl = tc::bf16x2_rn(hv[0] - __uint_as_float(hh << 16),
                                              hv[1] - __uint_as_float(hh & 0xFFFF0000u));
            *reinterpret_cast<uint32_t*>(xrow + off) = dh;
            *reinterpret_cast<uint32_t*>(xrow + 16384 + off) = dl;
            *reinterpret_cast<uint32_t*>(xrow + 32768 + off) = hh;
            *reinterpret_cast<uint32_t*>(xrow + 49152 + off) = hl;
          }
        }
        if constexpr (PLANES) {  // MMA4: D4 = dpre (W1 / 3), 3xTF32 as render_backward_pipe
          float d4v[16];
          zero(d4v);
          tc::wgmma_fence();
          mma4_mb(d4v, phi, plo, b4_hi, b4_lo);
          tc::wgmma_commit();
          tc::wgmma_wait<0>();
          tc::reg_fence(d4v);
          tc::store_frag_rows(d4v, d4s + 64 * mb * kD4Ld, kD4Ld, wig, lane);
        }
      }
      tc::fence_async_smem();
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(x_ready);
        if constexpr (PLANES) mbar_arrive(d4_full);
      }
    };
    if (total_steps > 0) act_fwd(0);
    for (uint32_t m = 0; m < total_steps; ++m) {
      if (m + 1 < total_steps) act_fwd(m + 1);
      act_bwd(m);
    }
  } else {
    // ================================ SHADING (forward and reverse) ================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::kShadeRegs));
    FieldConst fc;
    fc.A = p.n_attention;
    fc.use_sdf = p.use_sdf;
    const float beta = p.use_sdf ? p.beta[0] : 1.f;
    fc.inv_beta = p.use_sdf ? 1.f / beta : 0.f;
    fc.inv_alpha = p.use_sdf ? 1.f / p.alpha[0] : 0.f;
    float acc_b2[NOUT_PAD];
#pragma unroll
    for (int o = 0; o < NOUT_PAD; ++o) acc_b2[o] = 0.f;
    uint32_t m = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
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
      tc::bar_sync(1, kThreads);
      if (gt < 48)
        pal[gt] = (p.n_attention > 0 && gt < p.n_attention * 3)
                      ? p.palette[(size_t)b * p.n_attention * 3 + gt]
                      : 0.f;
      tc::bar_sync(1, kThreads);

      // upstream gradients of this ray (zero for padding lanes)
      const float vz = valid ? 1.f : 0.f;
      const float g_r = vz * g.g_rgb[ray * 3 + 0], g_g = vz * g.g_rgb[ray * 3 + 1],
                  g_b = vz * g.g_rgb[ray * 3 + 2];
      float g_m = (g.g_mask ? vz * g.g_mask[ray] : 0.f);
      const float out_m = g.out_mask[ray];
      float o_r = g.out_rgb[ray * 3 + 0], o_g = g.out_rgb[ray * 3 + 1],
            o_b = g.out_rgb[ray * 3 + 2];
      if (p.white_background) {
        g_m -= (g_r + g_g + g_b);
        const float bg = 1.f - out_m;
        o_r -= bg;
        o_g -= bg;
        o_b -= bg;
      }
      const float total = (g_r * o_r + g_g * o_g + g_b * o_b) + g_m * out_m;
      float accP[PLANES ? NA : 1];  // PLANES: palette / beta / alpha gradients of this ray
#pragma unroll
      for (int a = 0; a < (PLANES ? NA : 1); ++a) accP[a] = 0.f;
      float acc_beta = 0.f, acc_alpha = 0.f;

      MergeWalk mw;
      mw.init(p, r, ray, frac);
      float z = mw.pop();
      float T = 1.f, prefix = 0.f;
      for (int i = 0; i < n_total; ++i, ++m) {
        const bool has_next = (i + 1 < n_total);
        const float zn = has_next ? mw.pop() : z;
        const float delta = has_next ? (zn - z) * r.dn : 0.f;
        const uint32_t sl = m % kWgSlots, v = m / kWgSlots;
        float* const row = d2s + sl * (kThreads * kD2Ld) + gt * kD2Ld;  // D2 in, dOut out
        const float wx = r.ox + r.dx * z, wy = r.oy + r.dy * z, wz = r.oz + r.dz * z;
        const float x0 = wx * inv_range, x1 = wy * inv_range, x2 = wz * inv_range;
        const float keep = (fabsf(x0) > 1.f || fabsf(x1) > 1.f || fabsf(x2) > 1.f) ? 0.f : 1.f;
        NFI_STEP_WAIT(&d2_full[sl], v & 1);
        float o16[16];
#pragma unroll
        for (int o = 0; o < 16; ++o) o16[o] = row[o];
        float out[NOUT_PAD];
#pragma unroll
        for (int o = 0; o < NOUT_PAD; ++o) out[o] = o16[o] + b2s[o];
        // density (models/generator.py:629-636) and its derivative wrt out[0]
        float sigma, dsig_dout0, nd = 0.f, e_sdf = 0.f, sg = 0.f;
        if (fc.use_sdf) {
          nd = -out[0];
          e_sdf = tc::ex2_approx(-fabsf(nd) * (fc.inv_beta * kLog2e));
          sg = (nd > 0.f) ? 1.f : ((nd < 0.f) ? -1.f : 0.f);
          sigma = fc.inv_alpha * ((0.5f + 0.5f * sg * (1.f - e_sdf)) * keep);
          // analytic derivative also AT the zero crossing (see nfi_backward_pipe.cuh)
          dsig_dout0 = -(fc.inv_alpha * keep) * 0.5f * e_sdf * fc.inv_beta;
        } else {
          const float x = out[0] - 1.f;
          sigma = (x > 20.f ? x : log1pf(expf(x))) * keep;
          dsig_dout0 = keep * sigmoid_fast(x);
        }
        float probs[NA];
        float cr, cg, cb;
        if (fc.A > 0) {
          float mx = out[1];
#pragma unroll
          for (int a = 1; a < NA; ++a) mx = fmaxf(mx, out[1 + a]);
          float s = 0.f;
#pragma unroll
          for (int a = 0; a < NA; ++a) {
            probs[a] = tc::ex2_approx(out[1 + a] - mx);
            s += probs[a];
          }
          const float inv = __fdividef(1.f, s);
          cr = cg = cb = 0.f;
#pragma unroll
          for (int a = 0; a < NA; ++a) {
            probs[a] *= inv;
            cr = fmaf(probs[a], pal[3 * a + 0], cr);
            cg = fmaf(probs[a], pal[3 * a + 1], cg);
            cb = fmaf(probs[a], pal[3 * a + 2], cb);
          }
        } else {
          cr = sigmoid_fast(out[1]) * 2.004f - 1.002f;
          cg = sigmoid_fast(out[2]) * 2.004f - 1.002f;
          cb = sigmoid_fast(out[3]) * 2.004f - 1.002f;
#pragma unroll
          for (int a = 0; a < NA; ++a) probs[a] = 0.f;
        }
        // ---- compositing, forward and reverse (nfi_backward.cuh header)
        const float e_sd = __expf(-sigma * delta);
        const float a = 1.f - e_sd;
        const float w = a * T;
        const float s_i = (g_r * cr + g_g * cg + g_b * cb) + g_m;
        prefix = fmaf(w, s_i, prefix);
        const float one_m_a = 1.f - a;
        const float dsig = delta * one_m_a * (T * s_i - (total - prefix) / (one_m_a + 1e-10f));
        T = T * (one_m_a + 1e-10f);
        // ---- field head, reverse
        float dOut[16];
#pragma unroll
        for (int o = 0; o < 16; ++o) dOut[o] = 0.f;
        dOut[0] = dsig * dsig_dout0;
        if (PLANES && fc.use_sdf) {
          acc_beta = fmaf(dsig, fc.inv_alpha * keep * (-0.5f * sg * e_sdf * fabsf(nd) * fc.inv_beta *
                                                       fc.inv_beta), acc_beta);
          acc_alpha = fmaf(dsig, -sigma * fc.inv_alpha, acc_alpha);
        }
        const float wr = w * g_r, wg2 = w * g_g, wb = w * g_b;
        if (fc.A > 0) {
          float dp[NA];
          float dot = 0.f;
#pragma unroll
          for (int q = 0; q < NA; ++q) {
            const float vv = wr * pal[3 * q + 0] + wg2 * pal[3 * q + 1] + wb * pal[3 * q + 2];
            dp[q] = vv;
            dot = fmaf(probs[q], vv, dot);
            if (PLANES) accP[q] = fmaf(w, probs[q], accP[q]);
          }
#pragma unroll
          for (int q = 0; q < NA; ++q) dOut[1 + q] = probs[q] * (dp[q] - dot);
        } else {
          const float sr = (cr + 1.002f) / 2.004f, sg2 = (cg + 1.002f) / 2.004f,
                      sb = (cb + 1.002f) / 2.004f;
          dOut[1] = wr * 2.004f * sr * (1.f - sr);
          dOut[2] = wg2 * 2.004f * sg2 * (1.f - sg2);
          dOut[3] = wb * 2.004f * sb * (1.f - sb);
        }
#pragma unroll
        for (int o = 0; o < NOUT_PAD; ++o) acc_b2[o] += dOut[o];
        // ---- hand dOut to the tensor core: fp32 into the slot (MMA3), a bf16 hi/lo pair into
        //      the two [128][16] SWIZZLE_32B tiles the dW2 products read (once the previous
        //      step's chain has read them)
        {
#pragma unroll
          for (int o4 = 0; o4 < 4; ++o4)
            *reinterpret_cast<float4*>(row + 4 * o4) =
                make_float4(dOut[4 * o4], dOut[4 * o4 + 1], dOut[4 * o4 + 2], dOut[4 * o4 + 3]);
          NFI_STEP_WAIT(x_free, (m & 1) ^ 1);
          unsigned char* const et = base + Cfg::kSmE;
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            uint32_t eh[4], el[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float a0 = dOut[8 * q + 2 * i], a1 = dOut[8 * q + 2 * i + 1];
              eh[i] = tc::bf16x2_rn(a0, a1);
              el[i] = tc::bf16x2_rn(a0 - __uint_as_float(eh[i] << 16),
                                    a1 - __uint_as_float(eh[i] & 0xFFFF0000u));
            }
            const uint32_t off = tc::sw32_offset(gt, q);
            *reinterpret_cast<uint4*>(et + off) = make_uint4(eh[0], eh[1], eh[2], eh[3]);
            *reinterpret_cast<uint4*>(et + 4096 + off) = make_uint4(el[0], el[1], el[2], el[3]);
          }
          tc::fence_async_smem();
          __syncwarp();
          if (lane == 0) mbar_arrive(&dout_ready[sl]);
        }
        z = zn;
      }
      if constexpr (PLANES) {  // per-tile write-out, as render_backward_pipe
        if (g.grad_palette != nullptr && p.n_attention > 0) {
#pragma unroll
          for (int a = 0; a < NA; ++a) {
            const float pr = warp_sum(accP[a] * g_r), pg = warp_sum(accP[a] * g_g),
                        pb = warp_sum(accP[a] * g_b);
            if (lane == 0 && a < p.n_attention) {
              float* gp = g.grad_palette + ((size_t)b * p.n_attention + a) * 3;
              atomicAdd(gp + 0, pr);
              atomicAdd(gp + 1, pg);
              atomicAdd(gp + 2, pb);
            }
          }
        }
        if (p.use_sdf) {
          const float sb = warp_sum(acc_beta), sa = warp_sum(acc_alpha);
          if (lane == 0) {
            if (g.grad_beta) atomicAdd(g.grad_beta, sb);
            if (g.grad_alpha) atomicAdd(g.grad_alpha, sa);
          }
        }
      }
    }
    if (g.grad_b2 != nullptr) {
      const int nout = 1 + (p.n_attention > 0 ? p.n_attention : 3);
#pragma unroll
      for (int o = 0; o < NOUT_PAD; ++o) {
        const float sb = warp_sum(acc_b2[o]);
        if (lane == 0 && o < nout) atomicAdd(g.grad_b2 + o, sb);
      }
    }
  }
}

}  // namespace nfi
