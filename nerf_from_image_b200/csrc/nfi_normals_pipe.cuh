// Surface normals on the pipelined tensor-core path (SURVEY.md section 8f N3; run.py:229,
// models/generator.py:599-623, lib/nerf_utils.py:146-148): normal_map = sum_i w_i n_i (+ 1 - mask
// on a white background), n_i = normalize(grad_x sdf(x_i)), w_i the DETACHED compositing weights.
//
//   grad_x sdf = (dF/dx)^T (W1^T / 3) (W2[0,:] * sigmoid(pre))
//
// is what render_backward_pipe computes with dL/dpre replaced by s = W2[0,:] * sigmoid(pre): its
// MMA4 (D4 = s (W1 / 3)) and the texel re-read of its pose gradient (D4 . dF/dx per plane axis).
// This kernel is that kernel with the reverse compositing taken out: one sweep over the merged
// samples of a ray (fine depths from the forward pass's z_fine), gather -> MMA1 -> softplus ->
// MMA2 -> (shading: w_i) and -> s -> MMA4 -> (producers: re-read, dot, normalise, weight, sum).
// s needs nothing from the shading group, so the activation group issues all three GEMMs of a
// step back to back and releases the stage after layer 1.
// It runs after render_forward_pipe (which wrote z_fine and mask) and fills `normals`.
#pragma once
#include "nfi_backward_pipe.cuh"

namespace nfi {

template <int NOUT_PAD, int P>
__global__ void __launch_bounds__(BwdCfg<P>::kThreadsTotal, 1)
render_normals_pipe(const nfi_render_params p, const unsigned char* __restrict__ wimg,
                    const unsigned char* __restrict__ wimg_bwd) {
  constexpr bool CAM = true;
  using Cfg = BwdCfg<P>;
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
  uint64_t* a_free = full + NS;                 // [3] stage read by layer 1 (4 warps)
  uint64_t* d2_full = a_free + NS;              // [2] D2 in its slot (4 warps)
  uint64_t* dout_ready = d2_full + kBwdSlots;   // [2] D2 read, sample weight written (4 warps)
  uint64_t* d4_full = dout_ready + kBwdSlots;   // [2] D4 in its slot (4 warps)
  uint64_t* slot_free = d4_full + kBwdSlots;    // [2] D4 used (4 warps)
  uint64_t* wbar = slot_free + kBwdSlots;       // [2] weight images landed
  float* d2s = reinterpret_cast<float*>(base + Cfg::kSmD2);  // [2][128][kD2Ld]
  float* d4s = reinterpret_cast<float*>(base + Cfg::kSmD4);  // [2][128][kD4Ld]
  const float* b1s = reinterpret_cast<const float*>(base + kWiB1);
  const float* b2s = reinterpret_cast<const float*>(base + kWiB2);
  float* pal = reinterpret_cast<float*>(base + Cfg::kSmPal);
  float* frac = reinterpret_cast<float*>(base + Cfg::kSmFrac);
  if (tid < 128) frac[tid] = (float)tid / (float)S;
  float* wbuf = reinterpret_cast<float*>(base + Cfg::kSmBytes);   // [2 slots][128] sample weights
  float* w2r0 = wbuf + kBwdSlots * 128;                            // W2[0, :]
  if (tid < kHid) w2r0[tid] = p.w2[tid];

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
    tc::mbar_expect_tx(&wbar[0], kWiBytes);
    tc::tma_bulk_g2s(base, wimg, kWiBytes, &wbar[0]);
    tc::mbar_expect_tx(&wbar[1], kWbBytes);
    tc::tma_bulk_g2s(base + Cfg::kSmWb, wimg_bwd, kWbBytes, &wbar[1]);
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
      MergeWalk mw;
      mw.init(p, r, ray, frac);
      float an0 = 0.f, an1 = 0.f, an2 = 0.f;  // this set's share of sum_i w_i n_i

      // taps of the (up to) two steps this set has between "gathered" and "scattered"
      ByteTaps cur, nxt;
      uint32_t cur_in = 0, nxt_in = 0;  // interior flags, 2 bits per plane
      float cur_z = 0.f, nxt_z = 0.f;
      auto gather_step = [&](int i, const ByteTaps& tp) {
        const uint32_t m = n0 + (uint32_t)i;
        const uint32_t st = m % NS, u = m / NS;
        unsigned char* const stage = base + Cfg::kSmA + st * kPipeStageBytes;
        NFI_STEP_WAIT(&a_free[st], (u & 1) ^ 1);
        gather_to_tiles_lean(planes_b, R, tp, stage, stage + 16384, 32 * wig, lane);
        tc::fence_async_smem();
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
        NFI_STEP_WAIT(&dout_ready[sl], v & 1);  // the shading thread's weight of this sample
        const float wgt = wbuf[sl * 128 + 32 * wig + lane];
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
        if (lane == 0) mbar_arrive(&slot_free[sl]);  // (the sample weight was read before)
        {
          // grad_x sdf of this thread's sample (D4 carries the 1/3 of the plane mean already),
          // F.normalize (generator.py:620), weighted with the detached compositing weight
          const float nx = Gw[lane * 4 + 0] * inv_range, ny = Gw[lane * 4 + 1] * inv_range,
                      nz = Gw[lane * 4 + 2] * inv_range;
          const float inv = wgt / fmaxf(sqrtf((nx * nx + ny * ny) + nz * nz), 1e-12f);
          an0 = fmaf(nx, inv, an0);
          an1 = fmaf(ny, inv, an1);
          an2 = fmaf(nz, inv, an2);
        }
        __syncwarp();
        cur = nxt;
        cur_in = nxt_in;
        cur_z = nxt_z;
      }
      if (valid) {  // the two sets hold the odd / even steps: summed into the zeroed output
        float bg = 0.f;
        if (set == 0 && p.white_background) bg = 1.f - p.mask[ray];  // lib/nerf_utils.py:157-158
        atomicAdd(p.normals + ray * 3 + 0, an0 + bg);
        atomicAdd(p.normals + ray * 3 + 1, an1 + bg);
        atomicAdd(p.normals + ray * 3 + 2, an2 + bg);
      }
    }
  } else if (wg == 0) {
    // ================================ ACTIVATION: the three GEMMs ================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::kActRegs));
    const uint32_t base_s = tc::smem_u32(base);
    const uint64_t w1_hi = tc::gmma_desc_sw128(base_s + kWiW1Hi);
    const uint64_t w1_lo = tc::gmma_desc_sw128(base_s + kWiW1Lo);
    const uint64_t w2_hi = tc::gmma_desc_sw128(base_s + kWiW2Hi);
    const uint64_t w2_lo = tc::gmma_desc_sw128(base_s + kWiW2Lo);
    const uint64_t b4_hi = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kWbW1tHi);
    const uint64_t b4_lo = tc::gmma_desc_sw128(base_s + Cfg::kSmWb + kWbW1tLo);
    const uint64_t dsc_a0 = tc::gmma_desc_sw128(base_s + Cfg::kSmA);
    const int t = lane & 3;
    for (uint32_t m = 0; m < total_steps; ++m) {
      const uint32_t st = m % NS, u = m / NS, sl = m % kBwdSlots, v = m / kBwdSlots;
      const uint64_t dsc_a = dsc_a0 + (uint64_t)st * (kPipeStageBytes >> 4);
      float* d2 = d2s + sl * (kThreads * kD2Ld);
      float* d4 = d4s + sl * (kThreads * kD4Ld);
      NFI_STEP_WAIT(&full[st], u & 1);
      NFI_STEP_WAIT(&dout_ready[sl], (v & 1) ^ 1);  // D2 of step m - 2 read
      NFI_STEP_WAIT(&slot_free[sl], (v & 1) ^ 1);   // D4 of step m - 2 used
#pragma unroll 1
      for (int mb = 0; mb < 2; ++mb) {
        float d[32];
        zero(d);
        tc::wgmma_fence();
        tc::layer1_mb(d, dsc_a + mb * (8192 >> 4), dsc_a + ((16384 + mb * 8192) >> 4), w1_hi, w1_lo);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::reg_fence(d);
        if (mb == 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&a_free[st]);
        }
        {
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
        // d sdf / d pre_j = W2[0, j] sigmoid(pre_j),  sigmoid(pre) = 1 - 2^(-H log2 e)
        uint32_t shi[8][4], slo[8][4];
#pragma unroll
        for (int kb = 0; kb < 8; ++kb) {
          const float2 bb = *reinterpret_cast<const float2*>(b1s + 8 * kb + 2 * t);
          const float2 ww = *reinterpret_cast<const float2*>(w2r0 + 8 * kb + 2 * t);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float h = tc::softplus_mufu<true>(d[4 * kb + e] + ((e & 1) ? bb.y : bb.x));
            const float sg = 1.f - tc::ex2_approx(-h * kLog2e);
            tc::put_split(shi, slo, kb, tc::afrag_slot(e), ((e & 1) ? ww.y : ww.x) * sg);
          }
        }
        float d4v[16];
        zero(d4v);
        tc::wgmma_fence();
        mma4_mb(d4v, shi, slo, b4_hi, b4_lo);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::reg_fence(d4v);
        tc::store_frag_rows(d4v, d4 + 64 * mb * kD4Ld, kD4Ld, wig, lane);
      }
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&d2_full[sl]);
        mbar_arrive(&d4_full[sl]);
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

      MergeWalk mw;
      mw.init(p, r, ray, frac);
      float z = mw.pop();
      float T = 1.f;
      for (int i = 0; i < n_total; ++i, ++m) {
        const bool has_next = (i + 1 < n_total);
        const float zn = has_next ? mw.pop() : z;
        const float delta = has_next ? (zn - z) * r.dn : 0.f;
        const uint32_t sl = m % kBwdSlots, v = m / kBwdSlots;
        const float* row = d2s + sl * (kThreads * kD2Ld) + gt * kD2Ld;
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
        // density (models/generator.py:629-636) -> this sample's compositing weight
        float sigma;
        if (fc.use_sdf) {
          const float nd = -out[0];
          const float e_sdf = tc::ex2_approx(-fabsf(nd) * (fc.inv_beta * kLog2e));
          const float sg = (nd > 0.f) ? 1.f : ((nd < 0.f) ? -1.f : 0.f);
          sigma = fc.inv_alpha * ((0.5f + 0.5f * sg * (1.f - e_sdf)) * keep);
        } else {
          const float x = out[0] - 1.f;
          sigma = (x > 20.f ? x : log1pf(expf(x))) * keep;
        }
        const float a = 1.f - __expf(-sigma * delta);
        wbuf[sl * 128 + gt] = a * T;
        T = T * ((1.f - a) + 1e-10f);
        __syncwarp();
        if (lane == 0) mbar_arrive(&dout_ready[sl]);
        z = zn;
      }
    }
  }
}

}  // namespace nfi
