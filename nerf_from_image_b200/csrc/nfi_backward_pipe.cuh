// Backward render kernel, pipelined tensor-core variant (SURVEY.md section 8 row a13).
//
// Same mathematics as nfi_backward.cuh (single front-to-back sweep over the merged
// depth order, field re-evaluated at every sample, no saved per-sample tensor) but
// all four GEMMs of a sample step run on the tensor cores (wgmma) with 3xTF32 operands:
//
//   MMA1  D1 = F  W1^T          [128 x 32] x [32 x 64]   pre-activations (x log2 e)
//   MMA2  D2 = H  W2^T          [128 x 64] x [64 x 16]   decoder outputs
//   MMA3  D3 = dOut W2          [128 x 16] x [16 x 64]   dL/dH
//   MMA4  D4 = dpre (W1 / 3)    [128 x 64] x [64 x 32]   dL/d(texel features)
//
// Roles of the persistent CTA (one per SM, one 128-ray tile in flight), by warpgroup:
//   0..P-1  producer sets: set q gathers the steps n = q (mod P) exactly as the
//           forward kernel does and, when D4 of such a step is ready, scatters it
//           into the plane gradient (red.global.add.v4, 8 lanes per texel) and
//           accumulates the camera gradient of its rays;
//   P       shading, thread = ray: decoder outputs -> density / colour ->
//           reverse compositing -> dOut, palette / beta / alpha gradients;
//   P+1     activation: issues all four GEMMs (accumulators in its registers, one 64-row half
//           of the tile after the other) with softplus forward (D1 -> H) and its reverse
//           (D3, H -> dpre = D3 * (1 - exp(-H))) on the accumulator registers.  Its order is
//           fwd(m+1) before bwd(m), so that the shading chain of step m overlaps the forward
//           GEMMs of step m+1; bwd(m) recomputes D1 from the stage, which stays resident until
//           then (a stored H would not fit the shared memory).
// Shared-memory slots (two of each): D2 -> dOut ([128 x 20] fp32: the shading thread reads its
// row of D2 and writes its row of dOut in its place) and D4 ([128 x 36] fp32).
// Decoder-weight gradients (GAN generator step) are NOT produced here (nfi_wgrad_pipe.cuh).
#pragma once
#include "nfi_backward.cuh"  // red_add_v4
#include "nfi_forward_pipe.cuh"

namespace nfi {

constexpr int kBwdSlots = 2;
constexpr int kBwdStages = 3;
constexpr int kD4Ld = 36;  // floats per row of a D4 slot
constexpr int kD4SlotBytes = kThreads * kD4Ld * 4;
// backward weight image (bytes), appended to the forward image
constexpr int kWbW2tHi = 0;      // [64 rows = hidden j][32 k = output o, 16 used] SW128, 8 KB
constexpr int kWbW2tLo = 8192;
constexpr int kWbW1tHi = 16384;  // [32 rows = channel c][64 k = hidden j] as two [32 x 32] k-blocks
constexpr int kWbW1tLo = 24576;  //   (K positions in register-fragment order: tc::kpos_of_hidden)
constexpr int kWbBytes = 32768;
static_assert(kWbBytes == kBwdImageBytes, "backward weight image and its workspace slot");

// VD: the view-conditioned instantiation.  Its two weight images (nfi_layout.h) are larger, so its
// stages hold fp32 features (split into TF32 hi / lo in registers, as the forward kernel does)
// instead of hi / lo pairs, and it keeps the tile's view features and the rays' view-gradient sums
// (both in the activation warpgroup's fragment order) behind the D4 slots.  The offsets of the
// plain kernel do not depend on it.
template <int P, bool VD = false>
struct BwdCfg {
  static constexpr int kThreadsTotal = 256 + 128 * P;
  static constexpr int kSmWb = VD ? 41984 : 25600;         // backward weight image
  static constexpr int kSmA = kSmWb + (VD ? 41984 : kWbBytes);  // 58368 = 57 * 1024 (plain)
  static constexpr int kStageBytes = VD ? kFwdStageBytes : kPipeStageBytes;
  static constexpr int kSmD2 = kSmA + kBwdStages * kStageBytes;      // D2 / dOut slots
  static constexpr int kSmD4 = kSmD2 + kBwdSlots * kD2SlotBytes;     // D4 slots
  static constexpr int kSmView = kSmD4 + kBwdSlots * kD4SlotBytes;   // VD: view tile, then sums
  static constexpr int kSmVg = kSmView + (VD ? kViewTileBytes : 0);
  static constexpr int kSmStage = kSmVg + (VD ? kViewTileBytes : 0);  // per-warp coord-grad staging
  static constexpr int kStageWarp = 32 * 4 * 4;                      // [32][4] coord grads
  static constexpr int kSmPal = kSmStage + P * 4 * kStageWarp;
  static constexpr int kSmFrac = kSmPal + 48 * 4;
  static constexpr int kSmBars = kSmFrac + 128 * 4;
  // full[3], a_free[3], per slot: d2_full, dout_ready, d4_full, slot_free; weights x2
  static constexpr int kNumBars = 2 * kBwdStages + 4 * kBwdSlots + 2;
  static constexpr int kSmBytes = kSmBars + kNumBars * 8;
  // P = 2: 512 x 128 = 65536 = 128 x (144 + 112) + 256 x 128 (the producers keep the launch
  // allocation)
  static constexpr int kActRegs = 144;
  static constexpr int kShadeRegs = 112;
};

// dOut rows of one 64-row block (row-major slot, kD2Ld floats per row) as TF32 hi / lo register
// A fragments of the two k-blocks of K = 16
__device__ __forceinline__ void load_dout_frags(const float* rows, int warp, int lane,
                                                uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
  const int g = lane >> 2, t = lane & 3;
  const float* r0 = rows + (16 * warp + g) * kD2Ld + t;
#pragma unroll
  for (int kb = 0; kb < 2; ++kb) {
    tc::put_split(hi, lo, kb, 0, r0[8 * kb]);
    tc::put_split(hi, lo, kb, 1, r0[8 * kD2Ld + 8 * kb]);
    tc::put_split(hi, lo, kb, 2, r0[8 * kb + 4]);
    tc::put_split(hi, lo, kb, 3, r0[8 * kD2Ld + 8 * kb + 4]);
  }
}
// D3 = dOut_lo*B_hi + dOut_hi*B_lo + dOut_hi*B_hi   (K = 16: two k-steps), one 64-row block
__device__ __forceinline__ void mma3_mb(float (&d3)[32], const uint32_t (&hi)[2][4],
                                        const uint32_t (&lo)[2][4], uint64_t b_hi, uint64_t b_lo) {
  tc::wgmma_tf32_rs_n64(d3, lo[0], b_hi, 0);
  tc::wgmma_tf32_rs_n64(d3, lo[1], b_hi + 2, 1);
  tc::wgmma_tf32_rs_n64(d3, hi[0], b_lo, 1);
  tc::wgmma_tf32_rs_n64(d3, hi[1], b_lo + 2, 1);
  tc::wgmma_tf32_rs_n64(d3, hi[0], b_hi, 1);
  tc::wgmma_tf32_rs_n64(d3, hi[1], b_hi + 2, 1);
}
// VD: dG = dOut W3 (K = 16 outputs, N = 32 features), the same six products as mma3_mb
__device__ __forceinline__ void mma_dg_mb(float (&dg)[16], const uint32_t (&hi)[2][4],
                                          const uint32_t (&lo)[2][4], uint64_t b_hi, uint64_t b_lo) {
  tc::wgmma_tf32_rs_n32(dg, lo[0], b_hi, 0);
  tc::wgmma_tf32_rs_n32(dg, lo[1], b_hi + 2, 1);
  tc::wgmma_tf32_rs_n32(dg, hi[0], b_lo, 1);
  tc::wgmma_tf32_rs_n32(dg, hi[1], b_lo + 2, 1);
  tc::wgmma_tf32_rs_n32(dg, hi[0], b_hi, 1);
  tc::wgmma_tf32_rs_n32(dg, hi[1], b_hi + 2, 1);
}
// VD: D3 += dF W2[1..32] (K = 32 features, N = 64), dF as register fragments; D3 arrives holding
// the distance row's part
__device__ __forceinline__ void mma3_vd_mb(float (&d3)[32], const uint32_t (&hi)[4][4],
                                           const uint32_t (&lo)[4][4], uint64_t b_hi,
                                           uint64_t b_lo) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) tc::wgmma_tf32_rs_n64(d3, lo[ks], b_hi + 2 * ks, 1);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) tc::wgmma_tf32_rs_n64(d3, hi[ks], b_lo + 2 * ks, 1);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) tc::wgmma_tf32_rs_n64(d3, hi[ks], b_hi + 2 * ks, 1);
}
// D4 = dpre_lo*B_hi + dpre_hi*B_lo + dpre_hi*B_hi   (K = 64: two k-blocks of 4 k-steps)
__device__ __forceinline__ void mma4_mb(float (&d4)[16], const uint32_t (&hi)[8][4],
                                        const uint32_t (&lo)[8][4], uint64_t b_hi, uint64_t b_lo) {
#pragma unroll
  for (int ks = 0; ks < 8; ++ks)
    tc::wgmma_tf32_rs_n32(d4, lo[ks], b_hi + (ks >> 2) * 256 + (ks & 3) * 2, ks != 0);
#pragma unroll
  for (int ks = 0; ks < 8; ++ks)
    tc::wgmma_tf32_rs_n32(d4, hi[ks], b_lo + (ks >> 2) * 256 + (ks & 3) * 2, 1);
#pragma unroll
  for (int ks = 0; ks < 8; ++ks)
    tc::wgmma_tf32_rs_n32(d4, hi[ks], b_hi + (ks >> 2) * 256 + (ks & 3) * 2, 1);
}
template <int R>
__device__ __forceinline__ void zero(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) d[i] = 0.f;
}

// byte_taps plus the "gradient flows" flags of make_taps (coordinate strictly inside
// (0, R-1) BEFORE clamping): bit 0 x, bit 1 y.
__device__ __forceinline__ uint32_t byte_taps_in(float gx, float gy, int R, uint32_t plane_units,
                                                 uint32_t& o, float& fx, float& fy) {
  const float m = (float)(R - 1);
  const float ix = (gx + 1.f) * 0.5f * m;
  const float iy = (gy + 1.f) * 0.5f * m;
  byte_taps(gx, gy, R, plane_units, o, fx, fy);
  return ((ix > 0.f && ix < m) ? 1u : 0u) | ((iy > 0.f && iy < m) ? 2u : 0u);
}

// Sequential reader of a per-ray float array, four values per load.
struct Stream4 {
  const float4* base;
  float4 win;
  int blk;
  __device__ __forceinline__ void init(const float* p) {
    base = reinterpret_cast<const float4*>(p);
    blk = -1;
  }
  __device__ __forceinline__ float get(int i) {
    if ((i >> 2) != blk) {
      blk = i >> 2;
      win = __ldg(base + blk);
    }
    const int q = i & 3;
    return q == 0 ? win.x : (q == 1 ? win.y : (q == 2 ? win.z : win.w));
  }
};

// The merged depth order of one ray (run.py:283: stable sort of cat(coarse, fine)):
// coarse depths recomputed from near/far + jitter, fine depths read back from z_fine.
struct MergeWalk {
  Stream4 nz, zf;
  float tnear, tfar, jit;
  const float* frac;
  int S, c, k;
  bool fine, noisy;
  float ct, fz;
  __device__ __forceinline__ float coarse_t(int s) {
    return lerp_torch(tnear, tfar, frac[s]) + (noisy ? nz.get(s) : 0.f) * jit;
  }
  __device__ __forceinline__ void init(const nfi_render_params& p, const Ray& r, size_t ray,
                                       const float* frac_) {
    S = p.num_samples;
    fine = p.fine_sampling != 0;
    noisy = p.noise_mode == NFI_NOISE_EXPLICIT;
    tnear = r.tnear;
    tfar = r.tfar;
    jit = (r.tfar - r.tnear) / (float)S;
    frac = frac_;
    nz.init(noisy ? p.noise_t + ray * S : nullptr);
    zf.init(fine ? p.z_fine + ray * S : nullptr);
    c = k = 0;
    ct = coarse_t(0);
    fz = fine ? zf.get(0) : 0.f;
  }
  // next depth in merged order (ties: coarse first)
  __device__ __forceinline__ float pop() {
    const bool take_c = (c < S) && (!fine || k >= S || ct <= fz);
    float zz;
    if (take_c) {
      zz = ct;
      ++c;
      ct = (c < S) ? coarse_t(c) : 0.f;
    } else {
      zz = fz;
      ++k;
      fz = (k < S) ? zf.get(k) : 0.f;
    }
    return zz;
  }
};

// VD: the view-conditioned decoder.  `wimg` holds its forward image (nfi_layout.h) at 0 and its
// backward image at kVdBwdImageOffset.
template <int NOUT_PAD, int EXTRA, bool CAM, int P, bool VD = false>
__global__ void __launch_bounds__(BwdCfg<P>::kThreadsTotal, 1)
render_backward_pipe(const nfi_render_params p, const nfi_render_grads g,
                     const unsigned char* __restrict__ wimg) {
  using Cfg = BwdCfg<P, VD>;
  constexpr int kImgBytes = VD ? kVdBytes : kWiBytes;
  constexpr int kImgB1 = VD ? kVdB1 : kWiB1, kImgB2 = VD ? kVdHead : kWiB2;
  constexpr int kBwdImgOff = VD ? kVdBwdImageOffset : kBwdImageOffset;
  constexpr int kBwdImgBytes = VD ? kVbBytes : kWbBytes;
  constexpr int NA = NOUT_PAD - 1;
  constexpr int NS = kBwdStages;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* base = smem_raw;
  const int tid = threadIdx.x, lane = tid & 31;
  const int hw_wg = __shfl_sync(kFull, tid >> 7, 0);
  // logical role: 0 activation, 1 shading, 3.. producer sets (see nfi_forward_pipe.cuh)
  const int wg = (hw_wg < P) ? hw_wg + 3 : (P + 1 - hw_wg);
  const int gt = tid & 127;
  const int wig = __shfl_sync(kFull, gt >> 5, 0);
  const int S = p.num_samples;
  const int n_total = (p.fine_sampling ? 2 : 1) * S;  // steps per tile

  uint64_t* bars = reinterpret_cast<uint64_t*>(base + Cfg::kSmBars);
  uint64_t* full = bars;                        // [3] stage gathered (4 warps)
  uint64_t* a_free = full + NS;                 // [3] stage read by the last GEMM using it (4 warps)
  uint64_t* d2_full = a_free + NS;              // [2] D2 in its slot (4 warps)
  uint64_t* dout_ready = d2_full + kBwdSlots;   // [2] dOut in the same slot (4 warps)
  uint64_t* d4_full = dout_ready + kBwdSlots;   // [2] D4 in its slot (4 warps)
  uint64_t* slot_free = d4_full + kBwdSlots;    // [2] D4 scattered (4 warps)
  uint64_t* wbar = slot_free + kBwdSlots;       // [2] weight images landed
  float* d2s = reinterpret_cast<float*>(base + Cfg::kSmD2);  // [2][128][kD2Ld]
  float* d4s = reinterpret_cast<float*>(base + Cfg::kSmD4);  // [2][128][kD4Ld]
  const float* b1s = reinterpret_cast<const float*>(base + kImgB1);
  const float* b2s = reinterpret_cast<const float*>(base + kImgB2);
  float* pal = reinterpret_cast<float*>(base + Cfg::kSmPal);
  float* frac = reinterpret_cast<float*>(base + Cfg::kSmFrac);
  if (tid < 128) frac[tid] = (float)tid / (float)S;

  if (tid == 0) {
    if (tc::smem_u32(base) & 1023u) __trap();
    for (int i = 0; i < NS; ++i) {
      tc::mbar_init(&full[i], kWarps);
      tc::mbar_init(&a_free[i], kWarps);
    }
    for (int i = 0; i < kBwdSlots; ++i) {
      tc::mbar_init(&d2_full[i], kWarps);
      tc::mbar_init(&dout_ready[i], kWarps);
      tc::mbar_init(&d4_full[i], kWarps);
      tc::mbar_init(&slot_free[i], kWarps);
    }
    tc::mbar_init(&wbar[0], 1);
    tc::mbar_init(&wbar[1], 1);
    tc::fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    tc::mbar_expect_tx(&wbar[0], kImgBytes);
    tc::tma_bulk_g2s(base, wimg, kImgBytes, &wbar[0]);
    tc::mbar_expect_tx(&wbar[1], kBwdImgBytes);
    tc::tma_bulk_g2s(base + Cfg::kSmWb, wimg + kBwdImgOff, kBwdImgBytes, &wbar[1]);
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
    // ================================ PRODUCER / SCATTER ================================
    const int set = wg - 3;
    float* Gw = reinterpret_cast<float*>(base + Cfg::kSmStage + (set * 4 + wig) * Cfg::kStageWarp);
    const int q = lane >> 3, kq = lane & 7;
    const uint32_t row_units = (uint32_t)R * 8u;
    uint32_t n0 = 0;  // ring position of the tile's first step
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, n0 += (uint32_t)n_total) {
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
      const unsigned char* planes_b =
          reinterpret_cast<const unsigned char*>(p.planes) + (size_t)b * 3 * plane_bytes;
      float* gplanes_b = g.grad_planes ? g.grad_planes + (size_t)b * 3 * (plane_bytes >> 2) : nullptr;
      MergeWalk mw;
      mw.init(p, r, ray, frac);
      float gox = 0.f, goy = 0.f, goz = 0.f, gdx = 0.f, gdy = 0.f, gdz = 0.f;

      // taps of the (up to) two steps this set has between "gathered" and "scattered"
      ByteTaps cur, nxt;
      uint32_t cur_in = 0, nxt_in = 0;  // interior flags, 2 bits per plane
      float cur_z = 0.f, nxt_z = 0.f;
      auto gather_step = [&](int i, const ByteTaps& tp) {
        const uint32_t m = n0 + (uint32_t)i;
        const uint32_t st = m % NS, u = m / NS;
        unsigned char* const stage = base + Cfg::kSmA + st * Cfg::kStageBytes;
        NFI_STEP_WAIT(&a_free[st], (u & 1) ^ 1);
        if constexpr (VD) {  // fp32 stage, read with generic loads only
          gather_to_tiles_lean<TileStore::kFp32>(planes_b, R, tp, stage, nullptr, 32 * wig, lane);
        } else {
          gather_to_tiles_lean(planes_b, R, tp, stage, stage + 16384, 32 * wig, lane);
          tc::fence_async_smem();
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&full[st]);
      };
      // advance the merge walk to local step i and compute that sample's taps
      int walked = 0;
      auto prepare = [&](int i, ByteTaps& tp, uint32_t& in6, float& zz) {
        float z = 0.f;
        while (walked <= i) {
          z = mw.pop();
          ++walked;
        }
        zz = z;
        const float x0 = (r.ox + r.dx * z) * inv_range, x1 = (r.oy + r.dy * z) * inv_range,
                    x2 = (r.oz + r.dz * z) * inv_range;
        in6 = byte_taps_in(x0, x1, R, 0u, tp.o[0], tp.fx[0], tp.fy[0]);
        in6 |= byte_taps_in(x0, x2, R, plane_bytes >> 4, tp.o[1], tp.fx[1], tp.fy[1]) << 2;
        in6 |= byte_taps_in(x1, x2, R, plane_bytes >> 3, tp.o[2], tp.fx[2], tp.fy[2]) << 4;
      };
      if (set < n_total) {
        prepare(set, cur, cur_in, cur_z);
        gather_step(set, cur);
      }
      for (int i = set; i < n_total; i += P) {
        if (i + P < n_total) {
          prepare(i + P, nxt, nxt_in, nxt_z);
          gather_step(i + P, nxt);
        }
        // ---- scatter step i: D4 -> plane gradient (and camera gradient)
        const uint32_t m = n0 + (uint32_t)i;
        const uint32_t sl = m % kBwdSlots, v = m / kBwdSlots;
        // this warp's 32 rows of the D4 slot, read in place (released after the scatter)
        const float* Dw = d4s + sl * (kThreads * kD4Ld) + 32 * wig * kD4Ld;
        NFI_STEP_WAIT(&d4_full[sl], v & 1);
        if ((p.mlp_mode & 0x4000) && p.normals != nullptr && ray == (size_t)p.noise_seed && valid) {
          float* d32 = p.normals + (size_t)n_total * 8 + (size_t)i * 32;   // debug trace
#pragma unroll
          for (int k = 0; k < 32; ++k) d32[k] = Dw[lane * kD4Ld + k];
        }
        const ByteTaps& tp = cur;
#ifdef NFI_BWD_NO_SCATTER   // timing experiment: D4 is read and dropped
#pragma unroll 1
        for (int gq = 0; gq < 0; ++gq) {
#else
#pragma unroll 1
        for (int gq = 0; gq < 8; ++gq) {
#endif
          const int src = 4 * gq + q;
          const uint32_t in6 = CAM ? __shfl_sync(kFull, cur_in, src) : 0u;
          const float4 d4v = *reinterpret_cast<const float4*>(Dw + src * kD4Ld + 4 * kq);
          float gc0 = 0.f, gc1 = 0.f, gc2 = 0.f;
          // nw texel clamped to R-2: all four taps of a plane exist at fixed offsets
          const uint32_t dx = 8u;
          const uint32_t dy = row_units;
          uint32_t a00[3];
          float fxs[3], fys[3];
#pragma unroll
          for (int pl = 0; pl < 3; ++pl) {
            a00[pl] = __shfl_sync(kFull, tp.o[pl], src) | (uint32_t)kq;
            fxs[pl] = __shfl_sync(kFull, tp.fx[pl], src);
            fys[pl] = __shfl_sync(kFull, tp.fy[pl], src);
          }
          // Pose gradient: the twelve texel re-reads of this point group are issued back to back,
          // BEFORE the atomics (whose asm carries a memory clobber: a load written after one is
          // not hoisted above it, which left three dependent L2 round trips per group exposed).
          float4 v[3][4];
          if (CAM) {
#pragma unroll
            for (int pl = 0; pl < 3; ++pl) {
              v[pl][0] = ldg4(texel_ptr(planes_b, a00[pl]));
              v[pl][1] = ldg4(texel_ptr(planes_b, a00[pl] + dx));
              v[pl][2] = ldg4(texel_ptr(planes_b, a00[pl] + dy));
              v[pl][3] = ldg4(texel_ptr(planes_b, a00[pl] + dy + dx));
            }
          }
#ifdef NFI_BWD_NO_RED   // timing experiment: everything but the atomics themselves
          if (false) {
#else
          if (gplanes_b != nullptr) {
#endif
#pragma unroll
            for (int pl = 0; pl < 3; ++pl) {
              const float gx0 = 1.f - fxs[pl], gy0 = 1.f - fys[pl];
              const float w00 = gx0 * gy0, w01 = fxs[pl] * gy0, w10 = gx0 * fys[pl],
                          w11 = fxs[pl] * fys[pl];
              float* gp = gplanes_b;
              red_add_v4(gp + (size_t)a00[pl] * 4, d4v.x * w00, d4v.y * w00, d4v.z * w00,
                         d4v.w * w00);
              red_add_v4(gp + (size_t)(a00[pl] + dx) * 4, d4v.x * w01, d4v.y * w01, d4v.z * w01,
                         d4v.w * w01);
              red_add_v4(gp + (size_t)(a00[pl] + dy) * 4, d4v.x * w10, d4v.y * w10, d4v.z * w10,
                         d4v.w * w10);
              red_add_v4(gp + (size_t)(a00[pl] + dy + dx) * 4, d4v.x * w11, d4v.y * w11,
                         d4v.z * w11, d4v.w * w11);
            }
          }
          if (CAM) {
#pragma unroll
            for (int pl = 0; pl < 3; ++pl) {
              const float fx = fxs[pl], fy = fys[pl];
              const float gx0 = 1.f - fx, gy0 = 1.f - fy;
              const float4 v00 = v[pl][0], v01 = v[pl][1], v10 = v[pl][2], v11 = v[pl][3];
              // d/dix = (ne-nw)*gy0 + (se-sw)*gy1 ; d/diy = (sw-nw)*gx0 + (se-ne)*gx1
              float gx = 0.f, gy = 0.f;
#define NFI_ACC(cmp)                                                              \
  gx = fmaf(d4v.cmp, (v01.cmp - v00.cmp) * gy0 + (v11.cmp - v10.cmp) * fy, gx);    \
  gy = fmaf(d4v.cmp, (v10.cmp - v00.cmp) * gx0 + (v11.cmp - v01.cmp) * fx, gy);
              NFI_ACC(x) NFI_ACC(y) NFI_ACC(z) NFI_ACC(w)
#undef NFI_ACC
              // no gradient through a clamped coordinate (make_taps: inx / iny)
              const float mult = 0.5f * (float)(R - 1);
              const bool inx = (in6 >> (2 * pl)) & 1u, iny = (in6 >> (2 * pl + 1)) & 1u;
              gx = inx ? gx * mult : 0.f;
              gy = iny ? gy * mult : 0.f;
              if (pl == 0) { gc0 += gx; gc1 += gy; }
              else if (pl == 1) { gc0 += gx; gc2 += gy; }
              else { gc1 += gx; gc2 += gy; }
            }
          }
          if (CAM) {
#pragma unroll
            for (int o = 1; o < 8; o <<= 1) {
              gc0 += __shfl_xor_sync(kFull, gc0, o);
              gc1 += __shfl_xor_sync(kFull, gc1, o);
              gc2 += __shfl_xor_sync(kFull, gc2, o);
            }
            if (kq == 0) {
              Gw[src * 4 + 0] = gc0;
              Gw[src * 4 + 1] = gc1;
              Gw[src * 4 + 2] = gc2;
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&slot_free[sl]);
        if (CAM) {
          // D4 carries the 1/3 of the plane mean already
          const float dpx = Gw[lane * 4 + 0] * inv_range, dpy = Gw[lane * 4 + 1] * inv_range,
                      dpz = Gw[lane * 4 + 2] * inv_range;
          const float z = cur_z;
          gox += dpx; goy += dpy; goz += dpz;
          gdx = fmaf(dpx, z, gdx); gdy = fmaf(dpy, z, gdy); gdz = fmaf(dpz, z, gdz);
        }
        __syncwarp();
        cur = nxt;
        cur_in = nxt_in;
        cur_z = nxt_z;
      }
      if (CAM && valid && g.grad_origins != nullptr) {
        atomicAdd(g.grad_origins + ray * 3 + 0, gox);
        atomicAdd(g.grad_origins + ray * 3 + 1, goy);
        atomicAdd(g.grad_origins + ray * 3 + 2, goz);
        atomicAdd(g.grad_dirs + ray * 3 + 0, gdx);
        atomicAdd(g.grad_dirs + ray * 3 + 1, gdy);
        atomicAdd(g.grad_dirs + ray * 3 + 2, gdz);
      }
    }
  } else if (wg == 0) {
    // ================================ ACTIVATION: the four GEMMs ================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::kActRegs));
    const uint32_t base_s = tc::smem_u32(base);
    if constexpr (VD) {
    // Per step: fwd = the forward kernel's view-conditioned decoder (decoder_step_vd) from the
    // fp32 stage, which stays resident, keeping the leaky ReLU's branches (one bit per element,
    // 32 per thread); bwd, per 64-row half: D1 again from the stage, dG = dOut W3 (column 0 of W3
    // is zero: the distance's gradient does not leak in), dF = dG * (1 or 0.2) by the kept
    // branches, added to the ray's view-gradient sum, D3 = dF W2[1..32] + dDist W2[0], then dpre
    // and D4 as the plain kernel.
    const uint64_t w1_hi = tc::gmma_desc_sw128(base_s + kVdW1Hi);
    const uint64_t w1_lo = tc::gmma_desc_sw128(base_s + kVdW1Lo);
    const uint64_t w2_hi = tc::gmma_desc_sw128(base_s + kVdW2Hi);
    const uint64_t w2_lo = tc::gmma_desc_sw128(base_s + kVdW2Lo);
    const uint64_t w3_hi = tc::gmma_desc_sw128(base_s + kVdW3Hi);
    const uint64_t w3_lo = tc::gmma_desc_sw128(base_s + kVdW3Lo);
    const uint64_t g3_hi = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kVbW3Hi);
    const uint64_t g3_lo = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kVbW3Lo);
    const uint64_t b3_hi = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kVbW2tHi);
    const uint64_t b3_lo = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kVbW2tLo);
    const uint64_t b4_hi = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kVbW1tHi);
    const uint64_t b4_lo = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kVbW1tLo);
    const float* w2d = reinterpret_cast<const float*>(base + Cfg::kSmWb + kVbW2d);
    const float* b2f = reinterpret_cast<const float*>(base + kVdB2f);
    float4* vt = reinterpret_cast<float4*>(base + Cfg::kSmView) + gt;  // view tile (+ b2[1..32])
    float4* vg = reinterpret_cast<float4*>(base + Cfg::kSmVg) + gt;    // view-gradient sums
    const bool vgrad = g.grad_view_features != nullptr;
    const int t = lane & 3, gq = lane >> 2;
    auto clear_sums = [&]() {
      if (vgrad)
#pragma unroll
        for (int i = 0; i < 8; ++i) vg[i * kThreads] = make_float4(0.f, 0.f, 0.f, 0.f);
    };
    // the tile's sums -> grad_view_features (overwritten; rows outside the image skipped: they
    // carry the edge ray's view features but not its gradient)
    auto flush_sums = [&](int tile) {
      if (!vgrad) return;
      const TileCoord tcd = tile_coord(tile, tiles_x, tiles_y);
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = 64 * mb + 16 * wig + gq + 8 * h;
          int px, py;
          tile_pixel(tcd.tile_x, tcd.tile_y, row >> 5, row & 31, px, py);
          if (px >= p.width || py >= p.height) continue;
          const size_t ray = ((size_t)tcd.b * p.height + py) * p.width + px;
          float* dst = g.grad_view_features + ray * NFI_VIEW_FEATURES + 2 * t;
#pragma unroll
          for (int j = 0; j < NFI_VIEW_FEATURES / 8; ++j) {
            const float4 s = vg[(mb * 4 + j) * kThreads];
            *reinterpret_cast<float2*>(dst + 8 * j) = h ? make_float2(s.z, s.w) : make_float2(s.x, s.y);
          }
        }
      }
    };
    auto act_fwd = [&](uint32_t m) -> uint32_t {
      const uint32_t st = m % NS, u = m / NS, sl = m % kBwdSlots;
      NFI_STEP_WAIT(&full[st], u & 1);
      const uint32_t neg =
          decoder_step_vd(base + Cfg::kSmA + st * Cfg::kStageBytes, w1_hi, w1_lo, w2_hi, w2_lo,
                          w3_hi, w3_lo, b1s, vt, d2s + sl * (kThreads * kD2Ld), wig, lane, []() {});
      __syncwarp();
      if (lane == 0) mbar_arrive(&d2_full[sl]);
      return neg;
    };
    auto act_bwd = [&](uint32_t m, uint32_t neg) {
      const uint32_t st = m % NS, sl = m % kBwdSlots, v = m / kBwdSlots;
      const unsigned char* stage = base + Cfg::kSmA + st * Cfg::kStageBytes;
      const float* dout = d2s + sl * (kThreads * kD2Ld);
      float* d4 = d4s + sl * (kThreads * kD4Ld);
      NFI_STEP_WAIT(&dout_ready[sl], v & 1);
      NFI_STEP_WAIT(&slot_free[sl], (v & 1) ^ 1);  // D4 of step m - 2 scattered
#pragma unroll 1
      for (int mb = 0; mb < 2; ++mb) {
        uint32_t a_hi[4][4], a_lo[4][4];
        {
          float fa[4][4];
          tc::load_afrag_sw128(fa, stage, 64 * mb, wig, lane);
#pragma unroll
          for (int kb = 0; kb < 4; ++kb)
#pragma unroll
            for (int s = 0; s < 4; ++s) tc::put_split(a_hi, a_lo, kb, s, fa[kb][s]);
        }
        if (mb == 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&a_free[st]);
        }
        const float* drows = dout + 64 * mb * kD2Ld;
        float d[32], dg[16];
        zero(d);
        zero(dg);
        uint32_t ohi[2][4], olo[2][4];
        load_dout_frags(drows, wig, lane, ohi, olo);
        tc::wgmma_fence();
        tc::layer1_mb_rs(d, a_hi, a_lo, w1_hi, w1_lo);
        mma_dg_mb(dg, ohi, olo, g3_hi, g3_lo);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::reg_fence(d);
        tc::reg_fence(dg);
        // dF by the forward's branches, into the view-gradient sums and the A fragments of D3
        const uint32_t nb = neg >> (16 * mb);
        uint32_t fhi[4][4], flo[4][4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float df[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            df[e] = ((nb >> (4 * j + e)) & 1u) ? dg[4 * j + e] * 0.2f : dg[4 * j + e];
            tc::put_split(fhi, flo, j, tc::afrag_slot(e), df[e]);
          }
          if (vgrad) {
            float4 s = vg[(mb * 4 + j) * kThreads];
            s.x += df[0];
            s.y += df[1];
            s.z += df[2];
            s.w += df[3];
            vg[(mb * 4 + j) * kThreads] = s;
          }
        }
        // D3 starts from the distance row's part, dDist (column 0 of dOut) x w2 row 0
        float d3[32];
        {
          const float dd0 = drows[(16 * wig + gq) * kD2Ld], dd1 = drows[(16 * wig + gq + 8) * kD2Ld];
#pragma unroll
          for (int jb = 0; jb < 8; ++jb) {
            const float2 w = *reinterpret_cast<const float2*>(w2d + 8 * jb + 2 * t);
            d3[4 * jb + 0] = dd0 * w.x;
            d3[4 * jb + 1] = dd0 * w.y;
            d3[4 * jb + 2] = dd1 * w.x;
            d3[4 * jb + 3] = dd1 * w.y;
          }
        }
        tc::wgmma_fence();
        mma3_vd_mb(d3, fhi, flo, b3_hi, b3_lo);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::reg_fence(d3);
        uint32_t phi[8][4], plo[8][4];
#pragma unroll
        for (int kb = 0; kb < 8; ++kb) {
          const float2 bb = *reinterpret_cast<const float2*>(b1s + 8 * kb + 2 * t);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float h = tc::softplus_mufu<true>(d[4 * kb + e] + ((e & 1) ? bb.y : bb.x));
            const float sg = 1.f - tc::ex2_approx(-h * kLog2e);
            tc::put_split(phi, plo, kb, tc::afrag_slot(e), d3[4 * kb + e] * sg);
          }
        }
        float d4v[16];
        zero(d4v);
        tc::wgmma_fence();
        mma4_mb(d4v, phi, plo, b4_hi, b4_lo);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::reg_fence(d4v);
        tc::store_frag_rows(d4v, d4 + 64 * mb * kD4Ld, kD4Ld, wig, lane);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&d4_full[sl]);
    };
    // step m belongs to the CTA's tile m / n_total: its view tile is filled before the tile's
    // first fwd, its sums written after the tile's last bwd (the fwd of the next tile's first
    // step comes in between and only reads the view tile)
    clear_sums();
    uint32_t neg_cur = 0, neg_nxt = 0;
    if (total_steps > 0) {
      fill_view_tile(p, tile_coord(blockIdx.x, tiles_x, tiles_y), b2f, vt, wig, lane);
      neg_cur = act_fwd(0);
    }
    for (uint32_t m = 0; m < total_steps; ++m) {
      const int tile = (int)blockIdx.x + (int)(m / (uint32_t)n_total) * (int)gridDim.x;
      const bool last = (m + 1) % (uint32_t)n_total == 0;
      if (m + 1 < total_steps) {
        if (last)
          fill_view_tile(p, tile_coord(tile + (int)gridDim.x, tiles_x, tiles_y), b2f, vt, wig, lane);
        neg_nxt = act_fwd(m + 1);
      }
      act_bwd(m, neg_cur);
      neg_cur = neg_nxt;
      if (last) {
        flush_sums(tile);
        clear_sums();
      }
    }
    } else {
    const uint64_t w1_hi = tc::gmma_desc_sw128(base_s + kWiW1Hi);
    const uint64_t w1_lo = tc::gmma_desc_sw128(base_s + kWiW1Lo);
    const uint64_t w2_hi = tc::gmma_desc_sw128(base_s + kWiW2Hi);
    const uint64_t w2_lo = tc::gmma_desc_sw128(base_s + kWiW2Lo);
    const uint64_t b3_hi = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kWbW2tHi);
    const uint64_t b3_lo = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kWbW2tLo);
    const uint64_t b4_hi = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kWbW1tHi);
    const uint64_t b4_lo = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kWbW1tLo);
    const uint64_t dsc_a0 = tc::gmma_desc_sw128(base_s + Cfg::kSmA);
    const int t = lane & 3;
    // D1 -> softplus -> D2 into the slot
    auto act_fwd = [&](uint32_t m) {
      const uint32_t st = m % NS, u = m / NS, sl = m % kBwdSlots;
      NFI_STEP_WAIT(&full[st], u & 1);
      decoder_step(dsc_a0 + (uint64_t)st * (kPipeStageBytes >> 4), w1_hi, w1_lo, w2_hi, w2_lo, b1s,
                   d2s + sl * (kThreads * kD2Ld), wig, lane, []() {});
      __syncwarp();
      if (lane == 0) mbar_arrive(&d2_full[sl]);
    };
    // D1 again, D3 = dOut W2, dpre = D3 * sigmoid(pre), D4 = dpre (W1 / 3) into the slot
    //   sigmoid(pre) = 1 - exp(-softplus(pre)) = 1 - 2^(-H log2 e)
    auto act_bwd = [&](uint32_t m) {
      const uint32_t st = m % NS, sl = m % kBwdSlots, v = m / kBwdSlots;
      const uint64_t dsc_a = dsc_a0 + (uint64_t)st * (kPipeStageBytes >> 4);
      const float* dout = d2s + sl * (kThreads * kD2Ld);
      float* d4 = d4s + sl * (kThreads * kD4Ld);
      NFI_STEP_WAIT(&dout_ready[sl], v & 1);
      NFI_STEP_WAIT(&slot_free[sl], (v & 1) ^ 1);  // D4 of step m - 2 scattered
#pragma unroll 1
      for (int mb = 0; mb < 2; ++mb) {
        float d[32], d3[32];
        zero(d);
        zero(d3);
        uint32_t ohi[2][4], olo[2][4];
        load_dout_frags(dout + 64 * mb * kD2Ld, wig, lane, ohi, olo);
        tc::wgmma_fence();
        tc::layer1_mb(d, dsc_a + mb * (8192 >> 4), dsc_a + ((16384 + mb * 8192) >> 4), w1_hi, w1_lo);
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
          for (int e = 0; e < 4; ++e) {
            const float h = tc::softplus_mufu<true>(d[4 * kb + e] + ((e & 1) ? bb.y : bb.x));
            const float sg = 1.f - tc::ex2_approx(-h * kLog2e);
            tc::put_split(phi, plo, kb, tc::afrag_slot(e), d3[4 * kb + e] * sg);
          }
        }
        float d4v[16];
        zero(d4v);
        tc::wgmma_fence();
        mma4_mb(d4v, phi, plo, b4_hi, b4_lo);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::reg_fence(d4v);
        tc::store_frag_rows(d4v, d4 + 64 * mb * kD4Ld, kD4Ld, wig, lane);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&d4_full[sl]);
    };
    if (total_steps > 0) act_fwd(0);
    for (uint32_t m = 0; m < total_steps; ++m) {
      if (m + 1 < total_steps) act_fwd(m + 1);
      act_bwd(m);
    }
    }
  } else {
    // ================================ SHADING (forward and reverse) ================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::kShadeRegs));
    FieldConst fc;
    fc.A = p.n_attention;
    fc.use_sdf = p.use_sdf;
    const float beta = p.use_sdf ? p.beta[0] : 1.f;
    fc.inv_beta = p.use_sdf ? 1.f / beta : 0.f;
    fc.inv_alpha = p.use_sdf ? 1.f / p.alpha[0] : 0.f;
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
      float total = (g_r * o_r + g_g * o_g + g_b * o_b) + g_m * out_m;
      float ge0 = 0.f, ge1 = 0.f, ge2 = 0.f;
      if (EXTRA == 1 && g.g_extra != nullptr) {
        ge0 = vz * g.g_extra[ray * 3 + 0];
        ge1 = vz * g.g_extra[ray * 3 + 1];
        ge2 = vz * g.g_extra[ray * 3 + 2];
        total = fmaf(ge0, g.out_extra[ray * 3 + 0], total);
        total = fmaf(ge1, g.out_extra[ray * 3 + 1], total);
        total = fmaf(ge2, g.out_extra[ray * 3 + 2], total);
      }
      float accP[NA];
#pragma unroll
      for (int a = 0; a < NA; ++a) accP[a] = 0.f;
      float acc_beta = 0.f, acc_alpha = 0.f;
      float gox = 0.f, goy = 0.f, goz = 0.f, gdx = 0.f, gdy = 0.f, gdz = 0.f;  // coords output only

      MergeWalk mw;
      mw.init(p, r, ray, frac);
      float z = mw.pop();
      float T = 1.f, prefix = 0.f;
      for (int i = 0; i < n_total; ++i, ++m) {
        const bool has_next = (i + 1 < n_total);
        const float zn = has_next ? mw.pop() : z;
        const float delta = has_next ? (zn - z) * r.dn : 0.f;
        const uint32_t sl = m % kBwdSlots, v = m / kBwdSlots;
        float* const row = d2s + sl * (kThreads * kD2Ld) + gt * kD2Ld;  // D2 in, dOut out
        // ---- forward at this sample
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
        float sigma, dsig_dout0, e_sdf = 0.f, sg = 0.f, nd = 0.f;
        if (fc.use_sdf) {
          nd = -out[0];
          e_sdf = tc::ex2_approx(-fabsf(nd) * (fc.inv_beta * kLog2e));
          sg = (nd > 0.f) ? 1.f : ((nd < 0.f) ? -1.f : 0.f);
          sigma = fc.inv_alpha * ((0.5f + 0.5f * sg * (1.f - e_sdf)) * keep);
          // d cdf / d(-d) = e / (2 beta), also AT the zero crossing: autograd of the reference's
          // 0.5 + 0.5 sign(x)(1 - exp(-|x|/beta)) returns 0 for x == 0.0 exactly (sign(0) = 0),
          // which fp32 does produce (out[0] = D2 + b2 cancels to 0.0 on a few samples per
          // million); the analytic limit is used
          dsig_dout0 = -(fc.inv_alpha * keep) * 0.5f * e_sdf * fc.inv_beta;
        } else {
          const float x = out[0] - 1.f;
          sigma = (x > 20.f ? x : log1pf(expf(x))) * keep;
          dsig_dout0 = keep * sigmoid_fast(x);
        }
        // colour: softmax(logits) . palette (logits arrive in log2 units), or wide sigmoid
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
        float s_i = (g_r * cr + g_g * cg + g_b * cb) + g_m;
        if (EXTRA == 1) s_i += ge0 * wx + ge1 * wy + ge2 * wz;
        prefix = fmaf(w, s_i, prefix);
        const float one_m_a = 1.f - a;
        const float dsig = delta * one_m_a * (T * s_i - (total - prefix) / (one_m_a + 1e-10f));
        T = T * (one_m_a + 1e-10f);
        // ---- field head, reverse
        float dOut[16];
#pragma unroll
        for (int o = 0; o < 16; ++o) dOut[o] = 0.f;
        dOut[0] = dsig * dsig_dout0;
        if (fc.use_sdf) {
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
            // padded entries: probs = 0 (logit -1e30) and palette rows are zero
            const float vv = wr * pal[3 * q + 0] + wg2 * pal[3 * q + 1] + wb * pal[3 * q + 2];
            dp[q] = vv;
            dot = fmaf(probs[q], vv, dot);
            accP[q] = fmaf(w, probs[q], accP[q]);
          }
          // d/d(true logit); the forward logits were scaled by log2 e only inside ex2
#pragma unroll
          for (int q = 0; q < NA; ++q) dOut[1 + q] = probs[q] * (dp[q] - dot);
        } else {
          const float sr = (cr + 1.002f) / 2.004f, sg2 = (cg + 1.002f) / 2.004f,
                      sb = (cb + 1.002f) / 2.004f;
          dOut[1] = wr * 2.004f * sr * (1.f - sr);
          dOut[2] = wg2 * 2.004f * sg2 * (1.f - sg2);
          dOut[3] = wb * 2.004f * sb * (1.f - sb);
        }
        if ((p.mlp_mode & 0x4000) && p.normals != nullptr && ray == (size_t)p.noise_seed && valid) {
          float* q8 = p.normals + (size_t)i * 8;   // debug trace, see nfi_backward.cuh
          q8[0] = z; q8[1] = sigma; q8[2] = w; q8[3] = T; q8[4] = dsig; q8[5] = dOut[0];
          q8[6] = s_i; q8[7] = delta;
        }
        // ---- hand dOut to the tensor core (split into TF32 hi/lo by the activation group)
#pragma unroll
        for (int o4 = 0; o4 < 4; ++o4)
          *reinterpret_cast<float4*>(row + 4 * o4) =
              make_float4(dOut[4 * o4], dOut[4 * o4 + 1], dOut[4 * o4 + 2], dOut[4 * o4 + 3]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&dout_ready[sl]);
        if (EXTRA == 1) {  // coords output: d(w x)/dx = w
          const float dpx = w * ge0, dpy = w * ge1, dpz = w * ge2;
          gox += dpx; goy += dpy; goz += dpz;
          gdx = fmaf(dpx, z, gdx); gdy = fmaf(dpy, z, gdy); gdz = fmaf(dpz, z, gdz);
        }
        z = zn;
      }
      // ------------------------------------------------------------ write-out
      if (EXTRA == 1 && CAM && valid && g.grad_origins != nullptr) {
        atomicAdd(g.grad_origins + ray * 3 + 0, gox);
        atomicAdd(g.grad_origins + ray * 3 + 1, goy);
        atomicAdd(g.grad_origins + ray * 3 + 2, goz);
        atomicAdd(g.grad_dirs + ray * 3 + 0, gdx);
        atomicAdd(g.grad_dirs + ray * 3 + 1, gdy);
        atomicAdd(g.grad_dirs + ray * 3 + 2, gdz);
      }
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
}

}  // namespace nfi
