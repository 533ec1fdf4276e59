// Backward render kernel (SURVEY.md section 8 row a13), SIMT-MLP variant.
//
// Reverse mode of run.py:176-350 without any saved per-sample tensor: each
// thread walks its ray's samples once more in merged depth order (coarse
// depths recomputed from near/far + jitter, fine depths read back from the
// S floats per ray the forward pass kept) and, at every sample, re-evaluates
// the field, forms dL/dsigma_i and dL/drgb_i, and immediately back-propagates
// through the decoder and the bilinear fetch.
//
//   w_i = a_i T_i,  T_{i+1} = T_i (1 - a_i + 1e-10),  a_i = 1 - exp(-sigma_i d_i)
//   L   = sum_i w_i s_i,  s_i = g_rgb.c_i + g_mask' + g_extra.e_i
//   dL/dsigma_i = d_i (1-a_i) [ T_i s_i - (L - sum_{k<=i} w_k s_k)/(1-a_i+1e-10) ]
//
// The total L comes from the forward OUTPUTS (g . rgb_map etc.), which is what
// lets the sweep run front-to-back in a single pass.  What the reference
// treats as constants stays constant: near/far, all depths, the out-of-cube
// mask, depth_map (lib/nerf_utils.py:145, run.py:197,261; generator.py:605).
//
// Gradients leave the kernel as
//   planes   red.global.add.v4.f32 into a channel-last [B,3,R,R,32] buffer,
//            8 lanes per texel (the mirror image of the gather);
//   w1,b1,w2,b2,palette,beta,alpha   per-warp register/shared accumulators,
//            reduced per CTA and added once per CTA;
//   ray origin / unit direction      one float3 each per ray (the binding
//            chains them to tform_cam2world / focal with tiny torch ops).
#pragma once
#include "nfi_common.cuh"
#include "nfi_forward.cuh"  // kViewMlpPad, num_tiles

namespace nfi {

constexpr int kDRow = 68;  // padded row (floats) of the [32][64] staging tile

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b),
               "f"(c), "f"(d)
               : "memory");
}

__host__ __device__ inline size_t bwd_smem_floats(int nout_pad, bool wgrad, bool viewdir = false) {
  const int nm = viewdir ? kViewMlpPad : nout_pad;
  size_t n = kC * kHid + kHid + kHid * nm + nm + 48;  // weights, palette
  n += kWarps * 32 * kFRow;                                         // features / dF
  n += kWarps * 32 * 4;                                             // coord grads
  if (wgrad) n += kWarps * 32 * kDRow + kWarps * 32 * nm;           // staging
  if (wgrad) n += kC * kHid + kHid + kHid * nm + nm;                // CTA reduction
  if (viewdir) {
    n += kC * nout_pad + nout_pad + 2 * NFI_VIEW_FEATURES * kThreads;  // W3t, b3, x_ray, dx_ray
    if (wgrad) n += kC * nout_pad + nout_pad;                          // CTA reduction of dW3, db3
  }
  return n;
}

// VD: view-direction conditioning (nfi_forward.cuh); the head works on NOUT_PAD logits, the
// decoder's second layer on NM = 36 outputs.
template <int NOUT_PAD, bool WGRAD, bool VD = false>
__global__ void __launch_bounds__(kThreads)
render_backward_simt(const nfi_render_params p, const nfi_render_grads g) {
  constexpr int NA = NOUT_PAD - 1;
  constexpr int NM = VD ? kViewMlpPad : NOUT_PAD;
  extern __shared__ __align__(16) float smem_f[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int S = p.num_samples;
  const bool fine = p.fine_sampling != 0;
  const int nhead = 1 + (p.n_attention > 0 ? p.n_attention : 3);
  const int nout = VD ? 1 + NFI_VIEW_FEATURES : nhead;  // decoder (layer 2) outputs

  float* W1t = smem_f;                   // [32][64]
  float* b1s = W1t + kC * kHid;          // [64]
  float* W2t = b1s + kHid;               // [64][NM]
  float* b2s = W2t + kHid * NM;          // [NM]
  float* pal = b2s + NM;                 // [48]
  float* Fall = pal + 48;                // [4][32][kFRow]
  float* Gall = Fall + kWarps * 32 * kFRow;  // [4][32][4]
  float* Dall = Gall + kWarps * 32 * 4;      // [4][32][kDRow]   (WGRAD)
  float* Oall = Dall + (WGRAD ? kWarps * 32 * kDRow : 0);  // [4][32][NM]
  float* Racc = Oall + (WGRAD ? kWarps * 32 * NM : 0);  // CTA reduction
  constexpr int kRaccFloats = WGRAD ? kC * kHid + kHid + kHid * NM + NM : 0;
  float* W3t = Racc + kRaccFloats;             // [32][NOUT_PAD]   (VD)
  float* b3s = W3t + (VD ? kC * NOUT_PAD : 0);  // [NOUT_PAD]
  float* xs = b3s + (VD ? NOUT_PAD : 0);        // [32][128] mapper features, column = thread
  float* dxs = xs + (VD ? NFI_VIEW_FEATURES * kThreads : 0);  // [32][128] their gradient
  float* R3 = dxs + (VD ? NFI_VIEW_FEATURES * kThreads : 0);  // [NOUT_PAD][32] + [NOUT_PAD]  (VD && WGRAD)

  const int tiles_x = (p.width + kTileW - 1) / kTileW;
  const int tiles_y = (p.height + kTileH - 1) / kTileH;
  const int cta = blockIdx.x;
  const int b = cta / (tiles_x * tiles_y);
  const int trem = cta % (tiles_x * tiles_y);
  const int tile_y = trem / tiles_x, tile_x = trem % tiles_x;

  for (int i = tid; i < kC * kHid; i += kThreads) W1t[i] = p.w1[(i % kHid) * kC + i / kHid];
  for (int i = tid; i < kHid; i += kThreads) b1s[i] = p.b1[i];
  for (int i = tid; i < kHid * NM; i += kThreads) {
    const int j = i / NM, o = i % NM;
    W2t[i] = (o < nout) ? p.w2[o * kHid + j] : 0.f;
  }
  for (int i = tid; i < NM; i += kThreads) b2s[i] = (i < nout) ? p.b2[i] : 0.f;
  for (int i = tid; i < 48; i += kThreads)
    pal[i] = (p.n_attention > 0 && i < p.n_attention * 3)
                 ? p.palette[(size_t)b * p.n_attention * 3 + i]
                 : 0.f;
  if (WGRAD)
    for (int i = tid; i < kRaccFloats; i += kThreads) Racc[i] = 0.f;
  if (VD) {
    for (int i = tid; i < kC * NOUT_PAD; i += kThreads) {
      const int c = i / NOUT_PAD, o = i % NOUT_PAD;
      W3t[i] = (o >= 1 && o < nhead) ? p.w3[(o - 1) * NFI_VIEW_FEATURES + c] : 0.f;
    }
    for (int i = tid; i < NOUT_PAD; i += kThreads) b3s[i] = (i >= 1 && i < nhead) ? p.b3[i - 1] : 0.f;
    if (WGRAD)
      for (int i = tid; i < kC * NOUT_PAD + NOUT_PAD; i += kThreads) R3[i] = 0.f;
  }

  int px, py;
  tile_pixel(tile_x, tile_y, warp, lane, px, py);
  const bool valid = (px < p.width) && (py < p.height);
  px = min(px, p.width - 1);
  py = min(py, p.height - 1);
  const size_t ray = ((size_t)b * p.height + py) * p.width + px;
  if (VD) {
#pragma unroll
    for (int c4 = 0; c4 < NFI_VIEW_FEATURES / 4; ++c4) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(p.view_features +
                                                             ray * NFI_VIEW_FEATURES) + c4);
      xs[(4 * c4 + 0) * kThreads + tid] = v.x;
      xs[(4 * c4 + 1) * kThreads + tid] = v.y;
      xs[(4 * c4 + 2) * kThreads + tid] = v.z;
      xs[(4 * c4 + 3) * kThreads + tid] = v.w;
    }
#pragma unroll
    for (int c = 0; c < NFI_VIEW_FEATURES; ++c) dxs[c * kThreads + tid] = 0.f;
  }
  __syncthreads();

  Ray r;
  setup_ray(p, b, py, px, r);
  FieldConst fc;
  fc.A = p.n_attention;
  fc.use_sdf = p.use_sdf;
  const float beta = p.use_sdf ? p.beta[0] : 1.f;
  fc.inv_beta = p.use_sdf ? 1.f / beta : 0.f;
  fc.inv_alpha = p.use_sdf ? 1.f / p.alpha[0] : 0.f;

  const size_t plane_stride = (size_t)p.plane_res * p.plane_res * kC;
  const float* planes_b = p.planes + (size_t)b * 3 * plane_stride;
  float* gplanes_b = g.grad_planes ? g.grad_planes + (size_t)b * 3 * plane_stride : nullptr;
  const bool cam_grad = (g.grad_origins != nullptr);
  float* Fw = Fall + warp * 32 * kFRow;
  float* Gw = Gall + warp * 32 * 4;
  float* Dw = Dall + warp * 32 * kDRow;
  float* Ow = Oall + warp * 32 * NM;
  const float* frow = Fw + lane * kFRow;
  const bool explicit_noise = (p.noise_mode == NFI_NOISE_EXPLICIT);
  const int R = p.plane_res;

  // upstream gradients of this ray (zero for padding lanes)
  const float vz = valid ? 1.f : 0.f;
  const float g_r = vz * g.g_rgb[ray * 3 + 0], g_g = vz * g.g_rgb[ray * 3 + 1],
              g_b = vz * g.g_rgb[ray * 3 + 2];
  float g_m = (g.g_mask ? vz * g.g_mask[ray] : 0.f);
  const float out_m = g.out_mask[ray];
  float o_r = g.out_rgb[ray * 3 + 0], o_g = g.out_rgb[ray * 3 + 1], o_b = g.out_rgb[ray * 3 + 2];
  if (p.white_background) {
    g_m -= (g_r + g_g + g_b);
    const float bg = 1.f - out_m;
    o_r -= bg;
    o_g -= bg;
    o_b -= bg;
  }
  float total = (g_r * o_r + g_g * o_g + g_b * o_b) + g_m * out_m;
  float ge[NOUT_PAD];
#pragma unroll
  for (int a = 0; a < NOUT_PAD; ++a) ge[a] = 0.f;
  const int extra = (g.g_extra != nullptr) ? p.extra_mode : 0;
  if (extra != 0) {
    const int ne = (extra == NFI_EXTRA_COORDS) ? 3 : p.n_attention;
#pragma unroll
    for (int a = 0; a < NOUT_PAD; ++a)
      if (a < ne) {
        ge[a] = vz * g.g_extra[ray * ne + a];
        total = fmaf(ge[a], g.out_extra[ray * ne + a], total);
      }
  }

  // per-thread accumulators
  float acc_w1[WGRAD ? 64 : 1];  // dW1[j = 2*lane + (i>>5)][k = i&31]
  float acc_w2[WGRAD ? 2 * NM : 1];
  float acc_b1[2] = {0.f, 0.f};
  float acc_b2[(NM + 31) / 32] = {};  // output o = lane + 32 * i
  float acc_w3[(WGRAD && VD) ? NOUT_PAD : 1];  // dW3t[c = lane][o]
  float acc_b3 = 0.f;
  if (WGRAD) {
#pragma unroll
    for (int i = 0; i < 64; ++i) acc_w1[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 2 * NM; ++i) acc_w2[i] = 0.f;
    if (VD) {
#pragma unroll
      for (int i = 0; i < NOUT_PAD; ++i) acc_w3[i] = 0.f;
    }
  }
  float accP[NA];  // sum_i w_i probs_i  (-> palette gradient)
#pragma unroll
  for (int a = 0; a < NA; ++a) accP[a] = 0.f;
  float acc_beta = 0.f, acc_alpha = 0.f;
  float gox = 0.f, goy = 0.f, goz = 0.f, gdx = 0.f, gdy = 0.f, gdz = 0.f;

  const float span = r.tfar - r.tnear;
  auto coarse_t = [&](int s) {
    float t = lerp_torch(r.tnear, r.tfar, (float)s / (float)S);
    if (explicit_noise) t = t + p.noise_t[ray * S + s] * (span / (float)S);
    return t;
  };
  const int n_total = fine ? 2 * S : S;
  int c = 0, k = 0;
  float ct = coarse_t(0);
  float fz = fine ? p.z_fine[ray * S] : 0.f;
  // Pops the next depth in merged order (ties: coarse first, like a stable sort
  // of cat(coarse, fine), run.py:283).
  auto pop = [&]() -> float {
    const bool take_c = (c < S) && (!fine || k >= S || ct <= fz);
    float zz;
    if (take_c) {
      zz = ct;
      ++c;
      ct = (c < S) ? coarse_t(c) : 0.f;
    } else {
      zz = fz;
      ++k;
      fz = (k < S) ? p.z_fine[ray * S + k] : 0.f;
    }
    return zz;
  };
  float z = pop();
  float T = 1.f, prefix = 0.f;

  for (int i = 0; i < n_total; ++i) {
    const bool has_next = (i + 1 < n_total);
    const float zn = has_next ? pop() : z;
    const float delta = has_next ? (zn - z) * r.dn : 0.f;

    // ---- forward at this sample
    const float wx = r.ox + r.dx * z, wy = r.oy + r.dy * z, wz = r.oz + r.dz * z;
    const float x0 = wx / p.scene_range, x1 = wy / p.scene_range, x2 = wz / p.scene_range;
    const float keep = (fabsf(x0) > 1.f || fabsf(x1) > 1.f || fabsf(x2) > 1.f) ? 0.f : 1.f;
    gather_features(planes_b, R, x0, x1, x2, Fw, lane);
    float mo[NM];  // decoder outputs
    float h[kHid];
    mlp_forward<NM, true>(frow, W1t, b1s, W2t, b2s, mo, h);
    float out[NOUT_PAD];  // head inputs: distance-or-density, colour logits
    if constexpr (VD) {
      view_head<NOUT_PAD>(mo, xs + tid, W3t, b3s, out);
    } else {
#pragma unroll
      for (int o = 0; o < NOUT_PAD; ++o) out[o] = mo[o];
    }
    float sigma, cr, cg, cb;
    float probs[NOUT_PAD];
    field_head<NOUT_PAD>(out, fc, pal, keep, sigma, cr, cg, cb, probs);

    // ---- compositing, forward and reverse
    const float e_sd = expf(-sigma * delta);
    const float a = 1.f - e_sd;
    const float w = a * T;
    float s_i = (g_r * cr + g_g * cg + g_b * cb) + g_m;
    if (extra == NFI_EXTRA_COORDS) s_i += ge[0] * wx + ge[1] * wy + ge[2] * wz;
    if (extra == NFI_EXTRA_SEMANTICS) {
#pragma unroll
      for (int q = 0; q < NA; ++q) s_i = fmaf(ge[q], probs[q], s_i);
    }
    prefix = fmaf(w, s_i, prefix);
    const float one_m_a = 1.f - a;
    const float dsig = delta * one_m_a * (T * s_i - (total - prefix) / (one_m_a + 1e-10f));
    T = T * (one_m_a + 1e-10f);

    // ---- field head, reverse
    float dHd[NOUT_PAD];
#pragma unroll
    for (int o = 0; o < NOUT_PAD; ++o) dHd[o] = 0.f;
    if (fc.use_sdf) {
      const float nd = -out[0];
      const float e = expf(-fabsf(nd) * fc.inv_beta);
      const float sg = (nd > 0.f) ? 1.f : ((nd < 0.f) ? -1.f : 0.f);
      // sigma = inv_alpha * keep * (0.5 + 0.5 sg (1 - e))
      // (analytic derivative also at nd == 0.0 exactly, see nfi_backward_pipe.cuh)
      dHd[0] = dsig * (-(fc.inv_alpha * keep) * 0.5f * e * fc.inv_beta);
      acc_beta = fmaf(dsig, fc.inv_alpha * keep * (-0.5f * sg * e * fabsf(nd) * fc.inv_beta *
                                                   fc.inv_beta),
                      acc_beta);
      acc_alpha = fmaf(dsig, -sigma * fc.inv_alpha, acc_alpha);
    } else {
      dHd[0] = dsig * keep * sigmoid_fast(out[0] - 1.f);
    }
    const float wr = w * g_r, wg = w * g_g, wb = w * g_b;
    if (fc.A > 0) {
      float dp[NA];
      float dot = 0.f;
#pragma unroll
      for (int q = 0; q < NA; ++q) {
        float v = 0.f;
        if (q < fc.A) {
          v = wr * pal[3 * q + 0] + wg * pal[3 * q + 1] + wb * pal[3 * q + 2];
          if (extra == NFI_EXTRA_SEMANTICS) v = fmaf(w, ge[q], v);
        }
        dp[q] = v;
        dot = fmaf(probs[q], v, dot);
        accP[q] = fmaf(w, probs[q], accP[q]);
      }
#pragma unroll
      for (int q = 0; q < NA; ++q) dHd[1 + q] = probs[q] * (dp[q] - dot);
    } else {
      const float sr = (cr + 1.002f) / 2.004f, sg2 = (cg + 1.002f) / 2.004f,
                  sb = (cb + 1.002f) / 2.004f;
      dHd[1] = wr * 2.004f * sr * (1.f - sr);
      dHd[2] = wg * 2.004f * sg2 * (1.f - sg2);
      dHd[3] = wb * 2.004f * sb * (1.f - sb);
    }
    bool need = false;
#pragma unroll
    for (int o = 0; o < NOUT_PAD; ++o) need = need || (dHd[o] != 0.f);
    float dpx = 0.f, dpy = 0.f, dpz = 0.f;  // dL/d world point
    if (extra == NFI_EXTRA_COORDS) {
      dpx = w * ge[0];
      dpy = w * ge[1];
      dpz = w * ge[2];
    }
    __syncwarp();
    if (__any_sync(kFull, need)) {
      float dOut[NM];  // dL/d decoder outputs
      if constexpr (VD) {
        // ---- mapper closure, reverse: logits = b3 + W3 y, y = leaky_relu(x_ray + features)
        if (WGRAD) {
#pragma unroll
          for (int c = 0; c < NFI_VIEW_FEATURES; ++c) {
            const float zc = xs[c * kThreads + tid] + mo[1 + c];
            Dw[lane * kDRow + c] = zc > 0.f ? zc : zc * 0.2f;
          }
#pragma unroll
          for (int o = 0; o < NOUT_PAD; ++o) Dw[lane * kDRow + 32 + o] = dHd[o];
          __syncwarp();
          // dW3[o][c] += dlogit[pt][o] * y[pt][c]   (this lane: c = lane)
          for (int pt = 0; pt < 32; ++pt) {
            const float yv = Dw[pt * kDRow + lane];
#pragma unroll
            for (int o4 = 0; o4 < NOUT_PAD / 4; ++o4) {
              const float4 d4 = *reinterpret_cast<const float4*>(Dw + pt * kDRow + 32 + 4 * o4);
              acc_w3[4 * o4 + 0] = fmaf(d4.x, yv, acc_w3[4 * o4 + 0]);
              acc_w3[4 * o4 + 1] = fmaf(d4.y, yv, acc_w3[4 * o4 + 1]);
              acc_w3[4 * o4 + 2] = fmaf(d4.z, yv, acc_w3[4 * o4 + 2]);
              acc_w3[4 * o4 + 3] = fmaf(d4.w, yv, acc_w3[4 * o4 + 3]);
            }
            if (lane < NOUT_PAD) acc_b3 += Dw[pt * kDRow + 32 + lane];
          }
          __syncwarp();
        }
        dOut[0] = dHd[0];
#pragma unroll
        for (int o = 1 + NFI_VIEW_FEATURES; o < NM; ++o) dOut[o] = 0.f;
#pragma unroll
        for (int c = 0; c < NFI_VIEW_FEATURES; ++c) {
          const float4* wr3 = reinterpret_cast<const float4*>(W3t + c * NOUT_PAD);
          float dy = 0.f;
#pragma unroll
          for (int o4 = 0; o4 < NOUT_PAD / 4; ++o4) {
            const float4 wv = wr3[o4];  // column 0 is zero: dHd[0] does not leak in
            dy = fmaf(wv.x, dHd[4 * o4 + 0], dy);
            dy = fmaf(wv.y, dHd[4 * o4 + 1], dy);
            dy = fmaf(wv.z, dHd[4 * o4 + 2], dy);
            dy = fmaf(wv.w, dHd[4 * o4 + 3], dy);
          }
          const float zc = xs[c * kThreads + tid] + mo[1 + c];
          const float dz = zc > 0.f ? dy : dy * 0.2f;  // F.leaky_relu backward
          dOut[1 + c] = dz;
          dxs[c * kThreads + tid] += dz;
        }
      } else {
#pragma unroll
        for (int o = 0; o < NM; ++o) dOut[o] = dHd[o];
      }
      // ---- layer 2 reverse: dA_j, then dpre_j = dA_j * sigmoid(pre_j)
      if (WGRAD) {
#pragma unroll
        for (int j4 = 0; j4 < kHid / 4; ++j4) {
          float4 av;
          av.x = softplus_fast(h[4 * j4 + 0]);
          av.y = softplus_fast(h[4 * j4 + 1]);
          av.z = softplus_fast(h[4 * j4 + 2]);
          av.w = softplus_fast(h[4 * j4 + 3]);
          *reinterpret_cast<float4*>(Dw + lane * kDRow + 4 * j4) = av;
        }
#pragma unroll
        for (int o4 = 0; o4 < NM / 4; ++o4)
          *reinterpret_cast<float4*>(Ow + lane * NM + 4 * o4) =
              make_float4(dOut[4 * o4], dOut[4 * o4 + 1], dOut[4 * o4 + 2], dOut[4 * o4 + 3]);
        __syncwarp();
        // dW2[o][j] += dOut[pt][o] * a[pt][j]   (this lane: j = 2*lane, 2*lane+1)
        for (int pt = 0; pt < 32; ++pt) {
          const float2 aj = *reinterpret_cast<const float2*>(Dw + pt * kDRow + 2 * lane);
#pragma unroll
          for (int o4 = 0; o4 < NM / 4; ++o4) {
            const float4 d4 = *reinterpret_cast<const float4*>(Ow + pt * NM + 4 * o4);
            const float dv[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              acc_w2[4 * o4 + q] = fmaf(dv[q], aj.x, acc_w2[4 * o4 + q]);
              acc_w2[NM + 4 * o4 + q] = fmaf(dv[q], aj.y, acc_w2[NM + 4 * o4 + q]);
            }
          }
#pragma unroll
          for (int i = 0; i < (NM + 31) / 32; ++i)
            if (lane + 32 * i < NM) acc_b2[i] += Ow[pt * NM + lane + 32 * i];
        }
        __syncwarp();
      }
#pragma unroll
      for (int j = 0; j < kHid; ++j) {
        const float4* wrow = reinterpret_cast<const float4*>(W2t + j * NM);
        float dA = 0.f;
#pragma unroll
        for (int o4 = 0; o4 < NM / 4; ++o4) {
          const float4 wv = wrow[o4];
          dA = fmaf(wv.x, dOut[4 * o4 + 0], dA);
          dA = fmaf(wv.y, dOut[4 * o4 + 1], dA);
          dA = fmaf(wv.z, dOut[4 * o4 + 2], dA);
          dA = fmaf(wv.w, dOut[4 * o4 + 3], dA);
        }
        const float pre = h[j];
        h[j] = dA * (pre > 20.f ? 1.f : sigmoid_fast(pre));  // h now holds dpre
      }
      if (WGRAD) {
#pragma unroll
        for (int j4 = 0; j4 < kHid / 4; ++j4)
          *reinterpret_cast<float4*>(Dw + lane * kDRow + 4 * j4) =
              make_float4(h[4 * j4], h[4 * j4 + 1], h[4 * j4 + 2], h[4 * j4 + 3]);
        __syncwarp();
        // dW1[j][k] += dpre[pt][j] * f[pt][k]
        for (int pt = 0; pt < 32; ++pt) {
          const float2 dj = *reinterpret_cast<const float2*>(Dw + pt * kDRow + 2 * lane);
          acc_b1[0] += dj.x;
          acc_b1[1] += dj.y;
#pragma unroll
          for (int k4 = 0; k4 < kC / 4; ++k4) {
            const float4 f4 = *reinterpret_cast<const float4*>(Fw + pt * kFRow + 4 * k4);
            const float fv[4] = {f4.x, f4.y, f4.z, f4.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              acc_w1[4 * k4 + q] = fmaf(dj.x, fv[q], acc_w1[4 * k4 + q]);
              acc_w1[32 + 4 * k4 + q] = fmaf(dj.y, fv[q], acc_w1[32 + 4 * k4 + q]);
            }
          }
        }
      }
      __syncwarp();  // every lane is done reading features from Fw
      // ---- layer 1 reverse: dF_k = sum_j W1[j][k] dpre_j, written over Fw
#pragma unroll 1
      for (int k4 = 0; k4 < kC / 4; ++k4) {
        float df[4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const float4* wrow = reinterpret_cast<const float4*>(W1t + (4 * k4 + kk) * kHid);
          float acc = 0.f;
#pragma unroll
          for (int j4 = 0; j4 < kHid / 4; ++j4) {
            const float4 wv = wrow[j4];
            acc = fmaf(wv.x, h[4 * j4 + 0], acc);
            acc = fmaf(wv.y, h[4 * j4 + 1], acc);
            acc = fmaf(wv.z, h[4 * j4 + 2], acc);
            acc = fmaf(wv.w, h[4 * j4 + 3], acc);
          }
          df[kk] = acc * (1.f / 3.f);  // features are the mean of three planes
        }
        *reinterpret_cast<float4*>(Fw + lane * kFRow + 4 * k4) =
            make_float4(df[0], df[1], df[2], df[3]);
      }
      __syncwarp();
      // debug trace of one ray (tools/grad_trace.py): mlp_mode bit 0x4000, ray id in noise_seed,
      // buffer in p.normals: [n_total][8] scalars then [n_total][32] dL/d(feature)
      if ((p.mlp_mode & 0x4000) && p.normals != nullptr && ray == (size_t)p.noise_seed && valid) {
        float* q8 = p.normals + (size_t)i * 8;
        q8[0] = z; q8[1] = sigma; q8[2] = w; q8[3] = T; q8[4] = dsig; q8[5] = dHd[0];
        q8[6] = s_i; q8[7] = delta;
        float* d32 = p.normals + (size_t)n_total * 8 + (size_t)i * 32;
        for (int k = 0; k < 32; ++k) d32[k] = Fw[lane * kFRow + k];
      }
      // ---- bilinear fetch, reverse: 8 lanes per texel, vector reductions
      {
        const int q = lane >> 3, kq = lane & 7;
#pragma unroll 1
        for (int gi = 0; gi < 8; ++gi) {
          const int src = 4 * gi + q;
          const float c0 = __shfl_sync(kFull, x0, src);
          const float c1 = __shfl_sync(kFull, x1, src);
          const float c2 = __shfl_sync(kFull, x2, src);
          const float4 d4 = *reinterpret_cast<const float4*>(Fw + src * kFRow + 4 * kq);
          float gc0 = 0.f, gc1 = 0.f, gc2 = 0.f;
#pragma unroll
          for (int pl = 0; pl < 3; ++pl) {
            const float ga = (pl == 2) ? c1 : c0;
            const float gb = (pl == 0) ? c1 : c2;
            const Taps t = make_taps(ga, gb, R);
            if (gplanes_b != nullptr) {
              float* gp = gplanes_b + pl * plane_stride + 4 * kq;
              red_add_v4(gp + (size_t)t.o00 * kC, d4.x * t.w00, d4.y * t.w00, d4.z * t.w00,
                         d4.w * t.w00);
              red_add_v4(gp + (size_t)t.o01 * kC, d4.x * t.w01, d4.y * t.w01, d4.z * t.w01,
                         d4.w * t.w01);
              red_add_v4(gp + (size_t)t.o10 * kC, d4.x * t.w10, d4.y * t.w10, d4.z * t.w10,
                         d4.w * t.w10);
              red_add_v4(gp + (size_t)t.o11 * kC, d4.x * t.w11, d4.y * t.w11, d4.z * t.w11,
                         d4.w * t.w11);
            }
            if (cam_grad) {
              const float4* pp =
                  reinterpret_cast<const float4*>(planes_b + pl * plane_stride) + kq;
              const float4 v00 = ldg4(pp + (size_t)t.o00 * (kC / 4));
              const float4 v01 = ldg4(pp + (size_t)t.o01 * (kC / 4));
              const float4 v10 = ldg4(pp + (size_t)t.o10 * (kC / 4));
              const float4 v11 = ldg4(pp + (size_t)t.o11 * (kC / 4));
              // d/dix = (ne-nw)*gy0 + (se-sw)*gy1 ; d/diy = (sw-nw)*gx0 + (se-ne)*gx1
              float gx = 0.f, gy = 0.f;
#define NFI_ACC(cmp)                                                                     \
  gx = fmaf(d4.cmp, (v01.cmp - v00.cmp) * t.gy0 + (v11.cmp - v10.cmp) * t.gy1, gx);      \
  gy = fmaf(d4.cmp, (v10.cmp - v00.cmp) * t.gx0 + (v11.cmp - v01.cmp) * t.gx1, gy);
              NFI_ACC(x) NFI_ACC(y) NFI_ACC(z) NFI_ACC(w)
#undef NFI_ACC
              const float mult = 0.5f * (float)(R - 1);
              gx = t.inx ? gx * mult : 0.f;
              gy = t.iny ? gy * mult : 0.f;
              if (pl == 0) { gc0 += gx; gc1 += gy; }
              else if (pl == 1) { gc0 += gx; gc2 += gy; }
              else { gc1 += gx; gc2 += gy; }
            }
          }
          if (cam_grad) {
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
        if (cam_grad) {
          dpx += Gw[lane * 4 + 0] / p.scene_range;
          dpy += Gw[lane * 4 + 1] / p.scene_range;
          dpz += Gw[lane * 4 + 2] / p.scene_range;
        }
      }
    }
    // point = origin + dir * z
    gox += dpx; goy += dpy; goz += dpz;
    gdx = fmaf(dpx, z, gdx); gdy = fmaf(dpy, z, gdy); gdz = fmaf(dpz, z, gdz);
    __syncwarp();
    z = zn;
  }

  // ------------------------------------------------------------ write-out
  if (cam_grad && valid) {
    g.grad_origins[ray * 3 + 0] = gox;
    g.grad_origins[ray * 3 + 1] = goy;
    g.grad_origins[ray * 3 + 2] = goz;
    g.grad_dirs[ray * 3 + 0] = gdx;
    g.grad_dirs[ray * 3 + 1] = gdy;
    g.grad_dirs[ray * 3 + 2] = gdz;
  }
  if (g.grad_palette != nullptr && p.n_attention > 0) {
    // d rgb_map / d palette[a][c] = (sum_i w_i probs_i[a]) * g_c
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
  if (VD && valid && g.grad_view_features != nullptr) {
#pragma unroll
    for (int c4 = 0; c4 < NFI_VIEW_FEATURES / 4; ++c4)
      *reinterpret_cast<float4*>(g.grad_view_features + ray * NFI_VIEW_FEATURES + 4 * c4) =
          make_float4(dxs[(4 * c4 + 0) * kThreads + tid], dxs[(4 * c4 + 1) * kThreads + tid],
                      dxs[(4 * c4 + 2) * kThreads + tid], dxs[(4 * c4 + 3) * kThreads + tid]);
  }
  if (WGRAD) {
    // CTA-level reduction in shared memory, then one atomic per entry per CTA
    float* R1 = Racc;                       // [64][32]
    float* Rb1 = R1 + kC * kHid;            // [64]
    float* R2 = Rb1 + kHid;                 // [NM][64]
    float* Rb2 = R2 + kHid * NM;            // [NM]
#pragma unroll
    for (int i = 0; i < 64; ++i) atomicAdd(&R1[(2 * lane + (i >> 5)) * kC + (i & 31)], acc_w1[i]);
    atomicAdd(&Rb1[2 * lane], acc_b1[0]);
    atomicAdd(&Rb1[2 * lane + 1], acc_b1[1]);
#pragma unroll
    for (int o = 0; o < NM; ++o) {
      atomicAdd(&R2[o * kHid + 2 * lane], acc_w2[o]);
      atomicAdd(&R2[o * kHid + 2 * lane + 1], acc_w2[NM + o]);
    }
#pragma unroll
    for (int i = 0; i < (NM + 31) / 32; ++i)
      if (lane + 32 * i < NM) atomicAdd(&Rb2[lane + 32 * i], acc_b2[i]);
    if (VD) {
#pragma unroll
      for (int o = 0; o < NOUT_PAD; ++o) atomicAdd(&R3[o * kC + lane], acc_w3[o]);
      if (lane < NOUT_PAD) atomicAdd(&R3[kC * NOUT_PAD + lane], acc_b3);
    }
    __syncthreads();
    if (VD) {  // rows o = 1 .. nhead-1 of R3 are the logits a = o - 1
      if (g.grad_w3)
        for (int i = tid; i < (nhead - 1) * kC; i += kThreads) atomicAdd(g.grad_w3 + i, R3[kC + i]);
      if (g.grad_b3)
        for (int i = tid; i < nhead - 1; i += kThreads)
          atomicAdd(g.grad_b3 + i, R3[kC * NOUT_PAD + 1 + i]);
    }
    if (g.grad_w1)
      for (int i = tid; i < kC * kHid; i += kThreads) atomicAdd(g.grad_w1 + i, R1[i]);
    if (g.grad_b1)
      for (int i = tid; i < kHid; i += kThreads) atomicAdd(g.grad_b1 + i, Rb1[i]);
    if (g.grad_w2)
      for (int i = tid; i < nout * kHid; i += kThreads) atomicAdd(g.grad_w2 + i, R2[i]);
    if (g.grad_b2)
      for (int i = tid; i < nout; i += kThreads) atomicAdd(g.grad_b2 + i, Rb2[i]);
  }
}

namespace simt {

template <int NP, bool WG, bool VD>
int launch_bwd(const nfi_render_params& p, const nfi_render_grads& g, cudaStream_t st) {
  const size_t smem = bwd_smem_floats(NP, WG, VD) * sizeof(float);
  auto k = render_backward_simt<NP, WG, VD>;
  NFI_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k<<<(unsigned)num_tiles(p), kThreads, smem, st>>>(p, g);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace simt

// render_backward_simt, for arguments nfi_render_backward has checked.  nfi_render.cu instantiates
// it for VD = false, nfi_viewdir.cu for VD = true.
template <bool VD>
int launch_backward_simt(const nfi_render_params& p, const nfi_render_grads& g, cudaStream_t st) {
  const bool wg = g.grad_w1 || g.grad_b1 || g.grad_w2 || g.grad_b2 || g.grad_w3 || g.grad_b3;
  switch (nout_pad_of(p.n_attention)) {
    case 4: return wg ? simt::launch_bwd<4, true, VD>(p, g, st)
                      : simt::launch_bwd<4, false, VD>(p, g, st);
    case 12: return wg ? simt::launch_bwd<12, true, VD>(p, g, st)
                       : simt::launch_bwd<12, false, VD>(p, g, st);
    default: return wg ? simt::launch_bwd<16, true, VD>(p, g, st)
                       : simt::launch_bwd<16, false, VD>(p, g, st);
  }
}
extern template int launch_backward_simt<true>(const nfi_render_params&, const nfi_render_grads&,
                                               cudaStream_t);

}  // namespace nfi
