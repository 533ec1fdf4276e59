// Forward render kernel, SIMT-MLP variant (NFI_MLP_FP32_SIMT).
//
// One thread owns one ray for the whole of run.py:176-350; a CTA is a 16x8
// pixel tile of one image.  Per sample step a warp fetches its 32 points'
// tri-plane features cooperatively (nfi_common.cuh: gather_features), each
// thread runs the decoder on its own point, and the density->alpha product and
// colour sums stay in registers.  Nothing of size [rays x samples x features]
// is ever written to memory.  The only per-sample state that leaves registers
// is (t, sigma, rgb) of the S coarse samples -- needed again when the sorted
// union of coarse and fine samples is composited (run.py:283-335) -- which is
// parked in an L2-resident scratch slab, and two S-long per-ray columns in
// shared memory (coarse weights -> CDF, and the S fine depths).
#pragma once
#include "nfi_common.cuh"
#include "nfi_layout.h"

namespace nfi {

template <int NE, bool FAST = false>
struct Compositor {
  float T, ar, ag, ab, ad, am;
  float ae[NE > 0 ? NE : 1];
  float pz, ps, pr, pg, pb;
  float pe[NE > 0 ? NE : 1];
  bool have;

  __device__ __forceinline__ void init() {
    T = 1.f;
    ar = ag = ab = ad = am = 0.f;
#pragma unroll
    for (int e = 0; e < NE; ++e) ae[e] = 0.f;
    have = false;
    pz = ps = pr = pg = pb = 0.f;
  }
  // render_volume_density (lib/nerf_utils.py:135-150): the sample pushed LAST
  // is weighted once the NEXT one fixes its interval; the final sample has
  // delta = 0 and therefore weight 0.
  __device__ __forceinline__ void push(float z, float s, float r, float g, float b,
                                       const float* e, float dn) {
    if (have) {
      const float delta = (z - pz) * dn;
      const float a = 1.f - (FAST ? __expf(-ps * delta) : expf(-ps * delta));
      const float w = a * T;
      ar = fmaf(w, pr, ar);
      ag = fmaf(w, pg, ag);
      ab = fmaf(w, pb, ab);
      ad = fmaf(w, pz, ad);
      am += w;
#pragma unroll
      for (int i = 0; i < NE; ++i) ae[i] = fmaf(w, pe[i], ae[i]);
      T = T * ((1.f - a) + 1e-10f);
    }
    pz = z;
    ps = s;
    pr = r;
    pg = g;
    pb = b;
#pragma unroll
    for (int i = 0; i < NE; ++i) pe[i] = e[i];
    have = true;
  }
};

struct FwdSmem {
  float* W1t;  // [32][64]
  float* b1;   // [64]
  float* W2t;  // [64][NOUT_PAD]
  float* b2;   // [NOUT_PAD]
  float* pal;  // [16*3]
  float* F;    // [4][32][kFRow]
  float* G;    // [4][3][32][kFRow]  (normals only)
  float* colA; // [S][128]
  float* colB; // [S][128]
  float* W3t;  // [32][NOUT_PAD]  (view-direction conditioning only; column o = logit o-1)
  float* b3;   // [NOUT_PAD]
  float* xs;   // [32][128] per-ray mapper features, column = thread
};

constexpr int kViewMlpPad = 36;  // decoder outputs 1 + NFI_VIEW_FEATURES, padded to a float4 multiple

__host__ __device__ inline size_t fwd_smem_floats(int nout_pad, int S, bool fine,
                                                  bool normals = false, bool viewdir = false) {
  const int nm = viewdir ? kViewMlpPad : nout_pad;
  size_t n = kC * kHid + kHid + kHid * nm + nm + 48 + kWarps * 32 * kFRow;
  if (viewdir) n += kC * nout_pad + nout_pad + NFI_VIEW_FEATURES * kThreads;
  if (normals) n += kWarps * 3 * 32 * kFRow;  // d features / d coords, per warp
  if (fine) n += 2 * (size_t)S * kThreads;
  return n;
}

// scratch slab per CTA: float4 (sigma,r,g,b) [S][128], float t [S][128],
// float extra [S][NEs][128]
__host__ __device__ inline size_t fwd_scratch_floats_per_cta(int S, int ne_store) {
  return (size_t)S * kThreads * (5 + ne_store);
}

template <int NOUT_PAD>
__device__ __forceinline__ void load_weights_smem(const nfi_render_params& p, int b,
                                                  const FwdSmem& sm, int tid, int nout) {
  for (int i = tid; i < kC * kHid; i += kThreads) {
    const int k = i / kHid, j = i % kHid;
    sm.W1t[i] = p.w1[j * kC + k];
  }
  for (int i = tid; i < kHid; i += kThreads) sm.b1[i] = p.b1[i];
  for (int i = tid; i < kHid * NOUT_PAD; i += kThreads) {
    const int j = i / NOUT_PAD, o = i % NOUT_PAD;
    sm.W2t[i] = (o < nout) ? p.w2[o * kHid + j] : 0.f;
  }
  for (int i = tid; i < NOUT_PAD; i += kThreads) sm.b2[i] = (i < nout) ? p.b2[i] : 0.f;
  for (int i = tid; i < 48; i += kThreads)
    sm.pal[i] = (p.n_attention > 0 && i < p.n_attention * 3)
                    ? p.palette[(size_t)b * p.n_attention * 3 + i]
                    : 0.f;
}

// EXTRA: 0 none, 1 coords (3), 2 semantics (A).  NORM: also the composited surface normals
// (models/generator.py:599-623: normalised analytic gradient of the SDF with respect to the
// sample position; lib/nerf_utils.py:146-148: weighted with the detached weights), carried
// as three more "extras" after the EXTRA ones.
// VD: view-direction conditioning (--use_viewdir; models/generator.py:189-253,662-663): the
// decoder's second layer emits 1 + 32 values and the colour logits are
// w3 . leaky_relu(view_features[ray] + features, 0.2) + b3.
template <int NOUT_PAD, int EXTRA, bool FINE, bool NORM = false, bool VD = false>
__global__ void __launch_bounds__(kThreads)
render_forward_simt(const nfi_render_params p) {
  constexpr int NM = VD ? kViewMlpPad : NOUT_PAD;  // decoder (layer 2) outputs, padded
  constexpr int NE0 = (EXTRA == 0) ? 0 : (EXTRA == 1 ? 3 : NOUT_PAD - 1);
  constexpr int NE = NE0 + (NORM ? 3 : 0);
  constexpr int NES0 = (EXTRA == 2) ? NOUT_PAD - 1 : 0;
  constexpr int NES = NES0 + (NORM ? 3 : 0);  // extras parked in scratch
  extern __shared__ __align__(16) float smem_f[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int S = p.num_samples;

  FwdSmem sm;
  {
    float* q = smem_f;
    sm.W1t = q; q += kC * kHid;
    sm.b1 = q; q += kHid;
    sm.W2t = q; q += kHid * NM;
    sm.b2 = q; q += NM;
    sm.pal = q; q += 48;
    sm.W3t = q; q += VD ? kC * NOUT_PAD : 0;
    sm.b3 = q; q += VD ? NOUT_PAD : 0;
    sm.xs = q; q += VD ? NFI_VIEW_FEATURES * kThreads : 0;
    sm.F = q; q += kWarps * 32 * kFRow;
    sm.G = q; q += NORM ? kWarps * 3 * 32 * kFRow : 0;
    sm.colA = q; q += FINE ? (size_t)S * kThreads : 0;
    sm.colB = q;
  }
  const int tiles_x = (p.width + kTileW - 1) / kTileW;
  const int tiles_y = (p.height + kTileH - 1) / kTileH;
  const int cta = blockIdx.x;
  const int b = cta / (tiles_x * tiles_y);
  const int trem = cta % (tiles_x * tiles_y);
  const int tile_y = trem / tiles_x, tile_x = trem % tiles_x;

  const int nhead = 1 + (p.n_attention > 0 ? p.n_attention : 3);
  load_weights_smem<NM>(p, b, sm, tid, VD ? 1 + NFI_VIEW_FEATURES : nhead);
  if (VD) {
    for (int i = tid; i < kC * NOUT_PAD; i += kThreads) {
      const int c = i / NOUT_PAD, o = i % NOUT_PAD;
      sm.W3t[i] = (o >= 1 && o < nhead) ? p.w3[(o - 1) * NFI_VIEW_FEATURES + c] : 0.f;
    }
    for (int i = tid; i < NOUT_PAD; i += kThreads)
      sm.b3[i] = (i >= 1 && i < nhead) ? p.b3[i - 1] : 0.f;
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
      sm.xs[(4 * c4 + 0) * kThreads + tid] = v.x;
      sm.xs[(4 * c4 + 1) * kThreads + tid] = v.y;
      sm.xs[(4 * c4 + 2) * kThreads + tid] = v.z;
      sm.xs[(4 * c4 + 3) * kThreads + tid] = v.w;
    }
  }
  __syncthreads();

  Ray r;
  setup_ray(p, b, py, px, r);
  FieldConst fc;
  fc.A = p.n_attention;
  fc.use_sdf = p.use_sdf;
  fc.inv_beta = p.use_sdf ? 1.f / p.beta[0] : 0.f;
  fc.inv_alpha = p.use_sdf ? 1.f / p.alpha[0] : 0.f;

  const float* planes_b = p.planes + (size_t)b * 3 * p.plane_res * p.plane_res * kC;
  float* Fw = sm.F + warp * 32 * kFRow;
  const float* frow = Fw + lane * kFRow;
  const bool explicit_noise = (p.noise_mode == NFI_NOISE_EXPLICIT);

  float4* sc_srgb = nullptr;
  float* sc_t = nullptr;
  float* sc_e = nullptr;
  if (FINE) {
    float* slab = reinterpret_cast<float*>(p.workspace) +
                  (size_t)cta * fwd_scratch_floats_per_cta(S, NES);
    sc_srgb = reinterpret_cast<float4*>(slab);
    sc_t = slab + (size_t)4 * S * kThreads;
    sc_e = sc_t + (size_t)S * kThreads;
  }
  float* colA = sm.colA + tid;
  float* colB = sm.colB + tid;

  Compositor<NE> comp;
  comp.init();

  // Evaluates the field at depth t along this thread's ray (all 32 lanes of the
  // warp must call it together).
  auto eval = [&](float t, float& sigma, float& cr, float& cg, float& cb, float* ex) {
    const float wx = r.ox + r.dx * t, wy = r.oy + r.dy * t, wz = r.oz + r.dz * t;
    const float x0 = wx / p.scene_range, x1 = wy / p.scene_range, x2 = wz / p.scene_range;
    const float keep =
        (fabsf(x0) > 1.f || fabsf(x1) > 1.f || fabsf(x2) > 1.f) ? 0.f : 1.f;
    float out[NM];
    float h[kHid];
    if (NORM) {
      float* Gw = sm.G + warp * 3 * 32 * kFRow;
      gather_features_grad(planes_b, p.plane_res, x0, x1, x2, Fw, Gw, lane);
      mlp_forward<NM, true>(frow, sm.W1t, sm.b1, sm.W2t, sm.b2, out, h);  // h = pre-activations
      float n0, n1, n2;
      sdf_gradient<NM>(h, sm.W1t, sm.W2t, Gw, lane, n0, n1, n2);
      // common factors of the chain: (R-1)/2 per texel unit, 1/3 plane mean, 1/scene_range
      const float sc = 0.5f * (float)(p.plane_res - 1) / (3.f * p.scene_range);
      n0 *= sc;
      n1 *= sc;
      n2 *= sc;
      const float inv = 1.f / fmaxf(sqrtf((n0 * n0 + n1 * n1) + n2 * n2), 1e-12f);  // F.normalize
      ex[NE0 + 0] = n0 * inv;
      ex[NE0 + 1] = n1 * inv;
      ex[NE0 + 2] = n2 * inv;
    } else {
      gather_features(planes_b, p.plane_res, x0, x1, x2, Fw, lane);
      mlp_forward<NM, false>(frow, sm.W1t, sm.b1, sm.W2t, sm.b2, out, h);
    }
    __syncwarp();
    float probs[NOUT_PAD];
    if constexpr (VD) {
      float hd[NOUT_PAD];
      view_head<NOUT_PAD>(out, sm.xs + tid, sm.W3t, sm.b3, hd);
      field_head<NOUT_PAD>(hd, fc, sm.pal, keep, sigma, cr, cg, cb, probs);
    } else {
      field_head<NOUT_PAD>(out, fc, sm.pal, keep, sigma, cr, cg, cb, probs);
    }
    if (EXTRA == 1) {
      ex[0] = wx;
      ex[1] = wy;
      ex[2] = wz;
    } else if (EXTRA == 2) {
#pragma unroll
      for (int a = 0; a < NE0; ++a) ex[a] = probs[a];
    }
  };

  // ---------------- coarse pass (lib/nerf_utils.py:94-120) ----------------
  float wT = 1.f, prev_t = 0.f, prev_s = 0.f;
  const float span = r.tfar - r.tnear;
  for (int s = 0; s < S; ++s) {
    float t = lerp_torch(r.tnear, r.tfar, (float)s / (float)S);
    if (explicit_noise) t = t + p.noise_t[ray * S + s] * (span / (float)S);
    float sigma, cr, cg, cb;
    float ex[NE > 0 ? NE : 1];
    eval(t, sigma, cr, cg, cb, ex);
    if (FINE) {
      sc_srgb[s * kThreads + tid] = make_float4(sigma, cr, cg, cb);
      sc_t[s * kThreads + tid] = t;
#pragma unroll
      for (int a = 0; a < NES; ++a)
        sc_e[((size_t)s * NES + a) * kThreads + tid] = ex[a < NES0 ? a : NE0 + (a - NES0)];
      // render_volume_density_weights_only (lib/nerf_utils.py:164-180)
      if (s > 0) {
        const float delta = (t - prev_t) * r.dn;
        const float a = 1.f - expf(-prev_s * delta);
        colA[(s - 1) * kThreads] = a * wT;
        wT = wT * ((1.f - a) + 1e-10f);
      }
      prev_t = t;
      prev_s = sigma;
    } else {
      comp.push(t, sigma, cr, cg, cb, ex, r.dn);
    }
  }

  if (FINE) {
    colA[(S - 1) * kThreads] = 0.f;  // last interval is empty
    // ---- smoothing (run.py:266-272) + sample_pdf (lib/nerf_utils.py:183-222)
    // a[j] = 0.5*(max(w[j-1],w[j]) + max(w[j],w[j+1])) + 0.01 ; pdf over a[1..S-2]
    float sum = 0.f;
    {
      float wa = colA[0], wb = colA[kThreads], wc;
      for (int m = 0; m + 2 < S; ++m) {  // pw[m] = a[m+1] + 1e-5
        wc = colA[(m + 2) * kThreads];
        const float av = (fmaxf(wa, wb) + fmaxf(wb, wc)) * 0.5f + 0.01f;
        const float pw = av + 1e-5f;
        colB[m * kThreads] = pw;
        sum += pw;
        wa = wb;
        wb = wc;
      }
    }
    {
      float c = 0.f;
      colA[0] = 0.f;
      for (int m = 0; m + 2 < S; ++m) {
        c = c + colB[m * kThreads] / sum;
        colA[(m + 1) * kThreads] = c;  // cdf[0..S-2]
      }
    }
    // u -> colB, ascending
    if (explicit_noise) {
      for (int k = 0; k < S; ++k) {  // insertion sort (thread-private column)
        const float u = p.noise_u[ray * S + k];
        int i = k - 1;
        while (i >= 0 && colB[i * kThreads] > u) {
          colB[(i + 1) * kThreads] = colB[i * kThreads];
          --i;
        }
        colB[(i + 1) * kThreads] = u;
      }
    } else {
      for (int k = 0; k < S; ++k) colB[k * kThreads] = linspace01(k, S);
    }
    // inverse CDF, walking the (sorted) u's and the CDF together
    {
      int i = 1;
      const int last = S - 2;
      for (int k = 0; k < S; ++k) {
        const float u = colB[k * kThreads];
        while (i <= last && colA[i * kThreads] <= u) ++i;
        const int below = i - 1, above = min(last, i);
        const float c0 = colA[below * kThreads], c1 = colA[above * kThreads];
        const float z0 = 0.5f * (sc_t[(below + 1) * kThreads + tid] + sc_t[below * kThreads + tid]);
        const float z1 = 0.5f * (sc_t[(above + 1) * kThreads + tid] + sc_t[above * kThreads + tid]);
        float den = c1 - c0;
        if (den < 1e-5f) den = 1.f;
        const float tt = (u - c0) / den;
        colB[k * kThreads] = z0 + tt * (z1 - z0);
      }
    }
    if (p.z_fine != nullptr && valid)
      for (int k = 0; k < S; ++k) p.z_fine[ray * S + k] = colB[k * kThreads];

    // ------- fine pass + sorted merge + compositing (run.py:283-340) -------
    int c = 0;
    float ct = sc_t[tid];
    for (int k = 0; k < S; ++k) {
      const float z = colB[k * kThreads];
      float sigma, cr, cg, cb;
      float ex[NE > 0 ? NE : 1];
      eval(z, sigma, cr, cg, cb, ex);
      while (c < S && ct <= z) {
        const float4 q = sc_srgb[c * kThreads + tid];
        float ce[NE > 0 ? NE : 1];
        if (EXTRA == 1) {
          ce[0] = r.ox + r.dx * ct;
          ce[1] = r.oy + r.dy * ct;
          ce[2] = r.oz + r.dz * ct;
        }
#pragma unroll
        for (int a = 0; a < NES; ++a)
          ce[a < NES0 ? a : NE0 + (a - NES0)] = sc_e[((size_t)c * NES + a) * kThreads + tid];
        comp.push(ct, q.x, q.y, q.z, q.w, ce, r.dn);
        ++c;
        ct = (c < S) ? sc_t[c * kThreads + tid] : 0.f;
      }
      comp.push(z, sigma, cr, cg, cb, ex, r.dn);
    }
    while (c < S) {
      const float4 q = sc_srgb[c * kThreads + tid];
      float ce[NE > 0 ? NE : 1];
      if (EXTRA == 1) {
        ce[0] = r.ox + r.dx * ct;
        ce[1] = r.oy + r.dy * ct;
        ce[2] = r.oz + r.dz * ct;
      }
#pragma unroll
      for (int a = 0; a < NES; ++a)
        ce[a < NES0 ? a : NE0 + (a - NES0)] = sc_e[((size_t)c * NES + a) * kThreads + tid];
      comp.push(ct, q.x, q.y, q.z, q.w, ce, r.dn);
      ++c;
      ct = (c < S) ? sc_t[c * kThreads + tid] : 0.f;
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
    if (EXTRA != 0 && p.extra != nullptr) {
      const int ne_out = (EXTRA == 1) ? 3 : p.n_attention;
      for (int a = 0; a < NE0; ++a)
        if (a < ne_out) p.extra[ray * ne_out + a] = comp.ae[a];
    }
    if (NORM && p.normals != nullptr)  // lib/nerf_utils.py:157-158: white background applies too
      for (int a = 0; a < 3; ++a) p.normals[ray * 3 + a] = comp.ae[NE0 + a] + bg;
  }
}

// the SIMT kernels' grid: one CTA per 16 x 8 pixel tile
inline size_t num_tiles(const nfi_render_params& p) {
  const size_t tx = (p.width + kTileW - 1) / kTileW, ty = (p.height + kTileH - 1) / kTileH;
  return tx * ty * (size_t)p.batch;
}

namespace simt {

template <int NP, int EX, bool FINE, bool NORM, bool VD>
int launch_fwd(const nfi_render_params& p, size_t smem, cudaStream_t st) {
  if (smem > 227 * 1024)
    return fail("depth_samples_per_ray too large for the shared-memory columns");
  auto k = render_forward_simt<NP, EX, FINE, NORM, VD>;
  NFI_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k<<<(unsigned)num_tiles(p), kThreads, smem, st>>>(p);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

template <int NP, int EX, bool VD>
int fwd_fine(const nfi_render_params& p, bool normals, size_t smem, cudaStream_t st) {
  if (normals) {
    if (p.fine_sampling) return launch_fwd<NP, EX, true, true, VD>(p, smem, st);
    return launch_fwd<NP, EX, false, true, VD>(p, smem, st);
  }
  if (p.fine_sampling) return launch_fwd<NP, EX, true, false, VD>(p, smem, st);
  return launch_fwd<NP, EX, false, false, VD>(p, smem, st);
}

template <int NP, bool VD>
int fwd_extra(const nfi_render_params& p, bool normals, size_t smem, cudaStream_t st) {
  switch (p.extra_mode) {
    case NFI_EXTRA_COORDS: return fwd_fine<NP, 1, VD>(p, normals, smem, st);
    case NFI_EXTRA_SEMANTICS: return fwd_fine<NP, 2, VD>(p, normals, smem, st);
    default: return fwd_fine<NP, 0, VD>(p, normals, smem, st);
  }
}

}  // namespace simt

// render_forward_simt; `p.workspace` points at the scratch slabs (behind the weight-image header).
// nfi_render.cu instantiates it for VD = false, nfi_viewdir.cu for VD = true.
template <bool VD>
int launch_forward_simt(const nfi_render_params& p, bool normals, cudaStream_t st) {
  const int np = nout_pad_of(p.n_attention);
  const size_t smem =
      fwd_smem_floats(np, p.num_samples, p.fine_sampling != 0, normals, VD) * sizeof(float);
  switch (np) {
    case 4: return simt::fwd_extra<4, VD>(p, normals, smem, st);
    case 12: return simt::fwd_extra<12, VD>(p, normals, smem, st);
    default: return simt::fwd_extra<16, VD>(p, normals, smem, st);
  }
}
extern template int launch_forward_simt<true>(const nfi_render_params&, bool, cudaStream_t);

}  // namespace nfi
