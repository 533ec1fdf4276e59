// Shared device helpers for the fused tri-plane renderer (sm_90a).
//
// Everything here mirrors, stage by stage, the reference's per-ray render
// (citations into /root/reference).  The file is compiled with --fmad=false so
// that the per-ray geometry (a handful of operations per ray) rounds like the
// PyTorch elementwise kernels it replaces; the hot inner loops use explicit
// fmaf().
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "nfi_render.h"

namespace nfi {

constexpr int kC = NFI_PLANE_CHANNELS;  // 32 feature channels per plane
constexpr int kHid = NFI_HIDDEN;        // 64 hidden units
constexpr int kThreads = 128;           // rays per CTA (one thread = one ray)
constexpr int kWarps = kThreads / 32;
constexpr int kTileW = 16;              // CTA covers a 16x8 pixel tile:
constexpr int kTileH = 8;               // four 8x4 warp tiles, 2x2
constexpr int kFRow = 36;               // padded feature row (floats) in smem
constexpr unsigned kFull = 0xffffffffu;

struct Ray {
  float ox, oy, oz;  // origin
  float dx, dy, dz;  // unit direction
  float dn;          // |unit direction| as the reference recomputes it
  float tnear, tfar;
  bool hit;
};

// Pixel of this thread inside the CTA tile: warp w covers the 8x4 block at
// ((w&1)*8, (w>>1)*4); lane l is pixel (l&7, l>>3) of it.
__device__ __forceinline__ void tile_pixel(int tile_x, int tile_y, int warp, int lane, int& px,
                                           int& py) {
  px = tile_x * kTileW + (warp & 1) * 8 + (lane & 7);
  py = tile_y * kTileH + (warp >> 1) * 4 + (lane >> 3);
}

// get_ray_bundle + F.normalize + compute_near_far_planes
// (lib/nerf_utils.py:28-91, run.py:196, lib/nerf_utils.py:225-273).
// Rays that miss the cube do not get the global min/max fallback of :258-259:
// they never enter the cube, every sample is masked, outputs are background.
__device__ __forceinline__ void setup_ray(const nfi_render_params& p, int b, int py, int px,
                                          Ray& r) {
  float ii = (float)px / (float)p.width;
  // (row tiles: py counts from row_offset of a full_height-row image, nfi_render.h)
  float jj = (float)(py + p.row_offset) / (float)(p.full_height > 0 ? p.full_height : p.height);
  const float* M = p.c2w + b * 16;
  float rx, ry, rz;  // un-normalised direction
  if (p.focal != nullptr) {
    if (p.center != nullptr) {
      const float cx = p.center[b * 2 + 0], cy = p.center[b * 2 + 1];
      ii = ii - 0.5f * (2.f * cx - 1.f) - 0.5f;
      jj = jj - 0.5f * (2.f * cy - 1.f) - 0.5f;
    } else {
      ii = ii - 0.5f;
      jj = jj - 0.5f;
    }
    if (p.bbox != nullptr) {
      const float* bb = p.bbox + b * 4;  // [2][2]: row 0 start(x,y), row 1 range(x,y)
      ii = (bb[2] * (ii + 0.5f) + bb[0]) * 0.5f;
      jj = -((bb[3] * (-jj + 0.5f) + bb[1]) * 0.5f);
    }
    const float f = p.focal[b];
    ii = ii / f;
    jj = jj / f;
    const float cx = ii, cy = -jj, cz = -1.f;
    rx = (cx * M[0] + cy * M[1]) + cz * M[2];
    ry = (cx * M[4] + cy * M[5]) + cz * M[6];
    rz = (cx * M[8] + cy * M[9]) + cz * M[10];
    r.ox = M[3];
    r.oy = M[7];
    r.oz = M[11];
  } else {
    ii = (ii - 0.5f) * 2.f;
    jj = (jj - 0.5f) * 2.f;
    if (p.bbox != nullptr) {
      const float* bb = p.bbox + b * 4;
      ii = bb[2] * (ii / 2.f + 0.5f) + bb[0];
      jj = -(bb[3] * (-jj / 2.f + 0.5f) + bb[1]);
    }
    const float cx = ii, cy = -jj;
    r.ox = ((cx * M[0] + cy * M[1]) + 0.f * M[2]) + M[3];
    r.oy = ((cx * M[4] + cy * M[5]) + 0.f * M[6]) + M[7];
    r.oz = ((cx * M[8] + cy * M[9]) + 0.f * M[10]) + M[11];
    const float s = M[15];
    rx = -M[2] / s;
    ry = -M[6] / s;
    rz = -M[10] / s;
  }
  const float n = fmaxf(sqrtf((rx * rx + ry * ry) + rz * rz), 1e-12f);
  r.dx = rx / n;
  r.dy = ry / n;
  r.dz = rz / n;
  r.dn = sqrtf((r.dx * r.dx + r.dy * r.dy) + r.dz * r.dz);

  const float R = p.scene_range;
  const float ix = 1.f / r.dx, iy = 1.f / r.dy, iz = 1.f / r.dz;
  const float xlo = ((ix < 0.f ? R : -R) - r.ox) * ix, xhi = ((ix < 0.f ? -R : R) - r.ox) * ix;
  const float ylo = ((iy < 0.f ? R : -R) - r.oy) * iy, yhi = ((iy < 0.f ? -R : R) - r.oy) * iy;
  const float zlo = ((iz < 0.f ? R : -R) - r.oz) * iz, zhi = ((iz < 0.f ? -R : R) - r.oz) * iz;
  bool hit = !((xlo > yhi) || (ylo > xhi));
  float tn = fmaxf(xlo, ylo), tf = fminf(xhi, yhi);
  hit = hit && !((tn > zhi) || (zlo > tf));
  tn = fmaxf(tn, zlo);
  tf = fminf(tf, zhi);
  tn = fmaxf(tn, 0.1f);
  tf = fmaxf(tf, 0.1f);
  if (!((tf - tn) >= 1e-3f)) tf = tn + 1e-3f;
  r.tnear = tn;
  r.tfar = tf;
  r.hit = hit;
}

// torch.lerp(near, far, w)  (ATen: w < 0.5 ? a + w*(b-a) : b - (b-a)*(1-w))
__device__ __forceinline__ float lerp_torch(float a, float b, float w) {
  const float d = b - a;
  return (w < 0.5f) ? a + w * d : b - d * (1.f - w);
}

// torch.linspace(0, 1, S)[k]
__device__ __forceinline__ float linspace01(int k, int S) {
  const float step = 1.f / (float)(S - 1);
  return (k < S / 2) ? step * (float)k : 1.f - step * (float)(S - 1 - k);
}

// Bilinear taps of one plane, F.grid_sample(bilinear, border, align_corners=True)
// (models/generator.py:312-326; ATen GridSamplerKernel: unnormalise, clip, floor).
struct Taps {
  int o00, o01, o10, o11;      // texel offsets (in texels) of nw, ne, sw, se
  float w00, w01, w10, w11;    // their weights
  float gx0, gx1, gy0, gy1;    // 1-d weights (west/east, north/south) for d/dcoord
  bool inx, iny;               // coordinate strictly inside (0, R-1): grad flows
};

__device__ __forceinline__ Taps make_taps(float gx, float gy, int R) {
  Taps t;
  const float m = (float)(R - 1);
  float ix = ((gx + 1.f) / 2.f) * m;
  float iy = ((gy + 1.f) / 2.f) * m;
  t.inx = (ix > 0.f) && (ix < m);
  t.iny = (iy > 0.f) && (iy < m);
  ix = fminf(m, fmaxf(ix, 0.f));
  iy = fminf(m, fmaxf(iy, 0.f));
  const float fx = floorf(ix), fy = floorf(iy);
  t.gx1 = ix - fx;
  t.gx0 = (fx + 1.f) - ix;
  t.gy1 = iy - fy;
  t.gy0 = (fy + 1.f) - iy;
  const int x0 = (int)fx, y0 = (int)fy;
  const int x1 = min(x0 + 1, R - 1), y1 = min(y0 + 1, R - 1);
  t.o00 = y0 * R + x0;
  t.o01 = y0 * R + x1;
  t.o10 = y1 * R + x0;
  t.o11 = y1 * R + x1;
  t.w00 = t.gx0 * t.gy0;
  t.w01 = t.gx1 * t.gy0;
  t.w10 = t.gx0 * t.gy1;
  t.w11 = t.gx1 * t.gy1;
  return t;
}

__device__ __forceinline__ float4 ldg4(const float4* p) { return __ldg(p); }

__device__ __forceinline__ float4 bilerp4(const float4* plane, const Taps& t) {
  const float4 a = ldg4(plane + (size_t)t.o00 * (kC / 4));
  const float4 b = ldg4(plane + (size_t)t.o01 * (kC / 4));
  const float4 c = ldg4(plane + (size_t)t.o10 * (kC / 4));
  const float4 d = ldg4(plane + (size_t)t.o11 * (kC / 4));
  float4 e;
  e.x = fmaf(d.x, t.w11, fmaf(c.x, t.w10, fmaf(b.x, t.w01, a.x * t.w00)));
  e.y = fmaf(d.y, t.w11, fmaf(c.y, t.w10, fmaf(b.y, t.w01, a.y * t.w00)));
  e.z = fmaf(d.z, t.w11, fmaf(c.z, t.w10, fmaf(b.z, t.w01, a.z * t.w00)));
  e.w = fmaf(d.w, t.w11, fmaf(c.w, t.w10, fmaf(b.w, t.w01, a.w * t.w00)));
  return e;
}

// Warp-cooperative tri-plane fetch: 8 lanes read one 128-byte channel-last
// texel (float4 each), so a warp serves 4 points per iteration and each tap is
// exactly one cache line.  On return row `j` of `Frow` ([32][kFRow] floats in
// shared memory, private to this warp) holds the 32 mean-of-three-planes
// features of lane j's point (models/generator.py:328).
__device__ __forceinline__ void gather_features(const float* __restrict__ planes_b, int R,
                                                float x0, float x1, float x2, float* Frow,
                                                int lane) {
  const int q = lane >> 3, k = lane & 7;
  const size_t plane_stride = (size_t)R * R * kC;
#pragma unroll 2
  for (int g = 0; g < 8; ++g) {
    const int src = 4 * g + q;
    const float c0 = __shfl_sync(kFull, x0, src);
    const float c1 = __shfl_sync(kFull, x1, src);
    const float c2 = __shfl_sync(kFull, x2, src);
    const float4* base = reinterpret_cast<const float4*>(planes_b) + k;
    const float4 e0 = bilerp4(base, make_taps(c0, c1, R));
    const float4 e1 = bilerp4(base + plane_stride / 4, make_taps(c0, c2, R));
    const float4 e2 = bilerp4(base + 2 * (plane_stride / 4), make_taps(c1, c2, R));
    float4 f;
    f.x = ((e0.x + e1.x) + e2.x) / 3.f;
    f.y = ((e0.y + e1.y) + e2.y) / 3.f;
    f.z = ((e0.z + e1.z) + e2.z) / 3.f;
    f.w = ((e0.w + e1.w) + e2.w) / 3.f;
    *reinterpret_cast<float4*>(Frow + src * kFRow + 4 * k) = f;
  }
  __syncwarp();
}

// Bilinear interpolation plus its derivatives along the plane's two axes in TEXEL units
// (d/dix = (ne-nw) gy0 + (se-sw) gy1, d/diy = (sw-nw) gx0 + (se-ne) gx1; zero where
// the coordinate was clamped, as F.grid_sample's backward does).
__device__ __forceinline__ void bilerp4_grad(const float4* plane, const Taps& t, float4& e,
                                             float4& gx, float4& gy) {
  const float4 a = ldg4(plane + (size_t)t.o00 * (kC / 4));
  const float4 b = ldg4(plane + (size_t)t.o01 * (kC / 4));
  const float4 c = ldg4(plane + (size_t)t.o10 * (kC / 4));
  const float4 d = ldg4(plane + (size_t)t.o11 * (kC / 4));
  const float mx = t.inx ? 1.f : 0.f, my = t.iny ? 1.f : 0.f;
#define NFI_G(cmp)                                                                      \
  e.cmp = fmaf(d.cmp, t.w11, fmaf(c.cmp, t.w10, fmaf(b.cmp, t.w01, a.cmp * t.w00)));    \
  gx.cmp = ((b.cmp - a.cmp) * t.gy0 + (d.cmp - c.cmp) * t.gy1) * mx;                    \
  gy.cmp = ((c.cmp - a.cmp) * t.gx0 + (d.cmp - b.cmp) * t.gx1) * my;
  NFI_G(x) NFI_G(y) NFI_G(z) NFI_G(w)
#undef NFI_G
}

// gather_features plus the derivatives of the features with respect to the three
// normalised coordinates (rows of Grow: [3][32][kFRow]), up to the common factor
// (R-1)/2 / 3 the caller applies.  Plane xy sees (x0, x1), xz (x0, x2), yz (x1, x2).
__device__ __forceinline__ void gather_features_grad(const float* __restrict__ planes_b, int R,
                                                     float x0, float x1, float x2, float* Frow,
                                                     float* Grow, int lane) {
  const int q = lane >> 3, k = lane & 7;
  const size_t plane_stride = (size_t)R * R * kC;
#pragma unroll 1
  for (int g = 0; g < 8; ++g) {
    const int src = 4 * g + q;
    const float c0 = __shfl_sync(kFull, x0, src);
    const float c1 = __shfl_sync(kFull, x1, src);
    const float c2 = __shfl_sync(kFull, x2, src);
    const float4* base = reinterpret_cast<const float4*>(planes_b) + k;
    float4 e0, e1, e2, ax, ay, bx, by, cx, cy;
    bilerp4_grad(base, make_taps(c0, c1, R), e0, ax, ay);
    bilerp4_grad(base + plane_stride / 4, make_taps(c0, c2, R), e1, bx, by);
    bilerp4_grad(base + 2 * (plane_stride / 4), make_taps(c1, c2, R), e2, cx, cy);
    float4 f;
    f.x = ((e0.x + e1.x) + e2.x) / 3.f;
    f.y = ((e0.y + e1.y) + e2.y) / 3.f;
    f.z = ((e0.z + e1.z) + e2.z) / 3.f;
    f.w = ((e0.w + e1.w) + e2.w) / 3.f;
    *reinterpret_cast<float4*>(Frow + src * kFRow + 4 * k) = f;
    *reinterpret_cast<float4*>(Grow + src * kFRow + 4 * k) =
        make_float4(ax.x + bx.x, ax.y + bx.y, ax.z + bx.z, ax.w + bx.w);
    *reinterpret_cast<float4*>(Grow + (32 + src) * kFRow + 4 * k) =
        make_float4(ay.x + cx.x, ay.y + cx.y, ay.z + cx.z, ay.w + cx.w);
    *reinterpret_cast<float4*>(Grow + (64 + src) * kFRow + 4 * k) =
        make_float4(by.x + cy.x, by.y + cy.y, by.z + cy.z, by.w + cy.w);
  }
  __syncwarp();
}

// softplus as torch.nn.Softplus(beta=1, threshold=20): MUFU ex2 + lg2.
__device__ __forceinline__ float softplus_fast(float x) {
  const float e = __expf(-fabsf(x));
  const float s = fmaxf(x, 0.f) + __logf(1.f + e);
  return x > 20.f ? x : s;
}

// sigmoid(x) = d softplus / dx
__device__ __forceinline__ float sigmoid_fast(float x) {
  return __fdividef(1.f, 1.f + __expf(-x));
}

// Decoder MLP, one point per thread, fp32 FFMA (TriplanarDecoder.net,
// models/generator.py:294-299).  W1t is [32][64] (k-major), W2t is [64][NOUT_PAD],
// both in shared memory and read as warp-wide broadcasts.  `pre` (if KEEP)
// returns the 64 pre-activations for the backward pass.
template <int NOUT_PAD, bool KEEP>
__device__ __forceinline__ void mlp_forward(const float* __restrict__ frow,
                                            const float* __restrict__ W1t,
                                            const float* __restrict__ b1,
                                            const float* __restrict__ W2t,
                                            const float* __restrict__ b2, float (&out)[NOUT_PAD],
                                            float (&h)[kHid]) {
#pragma unroll
  for (int j4 = 0; j4 < kHid / 4; ++j4) {
    const float4 bv = *reinterpret_cast<const float4*>(b1 + 4 * j4);
    h[4 * j4 + 0] = bv.x;
    h[4 * j4 + 1] = bv.y;
    h[4 * j4 + 2] = bv.z;
    h[4 * j4 + 3] = bv.w;
  }
#pragma unroll 1
  for (int k4 = 0; k4 < kC / 4; ++k4) {
    const float4 f = *reinterpret_cast<const float4*>(frow + 4 * k4);
    const float fv[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const float4* wr = reinterpret_cast<const float4*>(W1t + (4 * k4 + kk) * kHid);
#pragma unroll
      for (int j4 = 0; j4 < kHid / 4; ++j4) {
        const float4 w = wr[j4];
        h[4 * j4 + 0] = fmaf(w.x, fv[kk], h[4 * j4 + 0]);
        h[4 * j4 + 1] = fmaf(w.y, fv[kk], h[4 * j4 + 1]);
        h[4 * j4 + 2] = fmaf(w.z, fv[kk], h[4 * j4 + 2]);
        h[4 * j4 + 3] = fmaf(w.w, fv[kk], h[4 * j4 + 3]);
      }
    }
  }
#pragma unroll
  for (int o4 = 0; o4 < NOUT_PAD / 4; ++o4) {
    const float4 bv = *reinterpret_cast<const float4*>(b2 + 4 * o4);
    out[4 * o4 + 0] = bv.x;
    out[4 * o4 + 1] = bv.y;
    out[4 * o4 + 2] = bv.z;
    out[4 * o4 + 3] = bv.w;
  }
#pragma unroll
  for (int j = 0; j < kHid; ++j) {
    const float a = softplus_fast(h[j]);
    if (!KEEP) h[j] = a;
    const float4* wr = reinterpret_cast<const float4*>(W2t + j * NOUT_PAD);
#pragma unroll
    for (int o4 = 0; o4 < NOUT_PAD / 4; ++o4) {
      const float4 w = wr[o4];
      out[4 * o4 + 0] = fmaf(w.x, a, out[4 * o4 + 0]);
      out[4 * o4 + 1] = fmaf(w.y, a, out[4 * o4 + 1]);
      out[4 * o4 + 2] = fmaf(w.z, a, out[4 * o4 + 2]);
      out[4 * o4 + 3] = fmaf(w.w, a, out[4 * o4 + 3]);
    }
  }
}

// d sdf / d(texel-unit coordinates) = W2[0,:] diag(sigmoid(pre)) W1 dF/dx  (analytic form of
// the autograd.grad call of models/generator.py:614-623).  `h` holds the 64 pre-activations on
// entry (mlp_forward<.., KEEP = true>) and is overwritten; Gw is this warp's
// gather_features_grad block.  The caller applies (R-1)/2 / 3 / scene_range.
template <int NOUT_PAD>
__device__ __forceinline__ void sdf_gradient(float (&h)[kHid], const float* __restrict__ W1t,
                                             const float* __restrict__ W2t,
                                             const float* __restrict__ Gw, int lane, float& n0,
                                             float& n1, float& n2) {
#pragma unroll
  for (int j = 0; j < kHid; ++j)
    h[j] = W2t[j * NOUT_PAD] * (h[j] > 20.f ? 1.f : 1.f / (1.f + expf(-h[j])));
  n0 = n1 = n2 = 0.f;
#pragma unroll 1
  for (int c = 0; c < kC; ++c) {
    const float4* wr = reinterpret_cast<const float4*>(W1t + c * kHid);
    float u = 0.f;
#pragma unroll
    for (int j4 = 0; j4 < kHid / 4; ++j4) {
      const float4 w = wr[j4];
      u = fmaf(w.x, h[4 * j4 + 0], u);
      u = fmaf(w.y, h[4 * j4 + 1], u);
      u = fmaf(w.z, h[4 * j4 + 2], u);
      u = fmaf(w.w, h[4 * j4 + 3], u);
    }
    n0 = fmaf(u, Gw[lane * kFRow + c], n0);
    n1 = fmaf(u, Gw[(32 + lane) * kFRow + c], n1);
    n2 = fmaf(u, Gw[(64 + lane) * kFRow + c], n2);
  }
}

// ViewDirectionMapper.mapper_closure (models/generator.py:242-251): colour logits from the
// decoder's 32 feature outputs and the ray's mapper features,
//   hd[1 + a] = b3[a] + sum_c w3[a][c] * leaky_relu(x_ray[c] + out[1 + c], 0.2),  hd[0] = out[0].
// `xcol` is this thread's column of the [32][kThreads] mapper-feature tile, W3t is [32][NOUT_PAD]
// with column 0 zero, b3s[0] = 0.
template <int NOUT_PAD, int NM>
__device__ __forceinline__ void view_head(const float (&out)[NM], const float* __restrict__ xcol,
                                          const float* __restrict__ W3t,
                                          const float* __restrict__ b3s, float (&hd)[NOUT_PAD]) {
#pragma unroll
  for (int o4 = 0; o4 < NOUT_PAD / 4; ++o4) {
    const float4 bv = *reinterpret_cast<const float4*>(b3s + 4 * o4);
    hd[4 * o4 + 0] = bv.x;
    hd[4 * o4 + 1] = bv.y;
    hd[4 * o4 + 2] = bv.z;
    hd[4 * o4 + 3] = bv.w;
  }
#pragma unroll
  for (int c = 0; c < NFI_VIEW_FEATURES; ++c) {
    const float z = xcol[c * kThreads] + out[1 + c];
    const float y = z > 0.f ? z : z * 0.2f;
    const float4* wr = reinterpret_cast<const float4*>(W3t + c * NOUT_PAD);
#pragma unroll
    for (int o4 = 0; o4 < NOUT_PAD / 4; ++o4) {
      const float4 w = wr[o4];
      hd[4 * o4 + 0] = fmaf(w.x, y, hd[4 * o4 + 0]);
      hd[4 * o4 + 1] = fmaf(w.y, y, hd[4 * o4 + 1]);
      hd[4 * o4 + 2] = fmaf(w.z, y, hd[4 * o4 + 2]);
      hd[4 * o4 + 3] = fmaf(w.w, y, hd[4 * o4 + 3]);
    }
  }
  hd[0] = out[0];
}

// Density and colour from the decoder outputs (models/generator.py:625-679).
struct FieldConst {
  float inv_beta;   // 1 / beta
  float inv_alpha;  // 1 / alpha
  int A;            // palette entries (0: direct wide-sigmoid colour)
  int use_sdf;
};

template <int NOUT_PAD, bool FAST = false>
__device__ __forceinline__ void field_head(const float (&out)[NOUT_PAD], const FieldConst& fc,
                                           const float* __restrict__ pal /*smem [A][3]*/,
                                           float keep /*1 - outside*/, float& sigma, float& cr,
                                           float& cg, float& cb, float (&probs)[NOUT_PAD]) {
  const float d = out[0];
  if (fc.use_sdf) {
    const float nd = -d;
    const float e = FAST ? __expf(-fabsf(nd) * fc.inv_beta) : expf(-fabsf(nd) * fc.inv_beta);
    const float sg = (nd > 0.f) ? 1.f : ((nd < 0.f) ? -1.f : 0.f);
    const float cdf = 0.5f + 0.5f * sg * (1.f - e);
    sigma = fc.inv_alpha * (cdf * keep);
  } else {
    const float x = d - 1.f;
    sigma = (x > 20.f ? x : log1pf(expf(x))) * keep;
  }
  if (fc.A > 0) {
    float m = -INFINITY;
#pragma unroll
    for (int a = 0; a < NOUT_PAD - 1; ++a)
      if (a < fc.A) m = fmaxf(m, out[1 + a]);
    float s = 0.f;
#pragma unroll
    for (int a = 0; a < NOUT_PAD - 1; ++a) {
      const float e = (a < fc.A) ? __expf(out[1 + a] - m) : 0.f;
      probs[a] = e;
      s += e;
    }
    const float inv = FAST ? __fdividef(1.f, s) : 1.f / s;
    cr = cg = cb = 0.f;
#pragma unroll
    for (int a = 0; a < NOUT_PAD - 1; ++a) {
      probs[a] *= inv;
      if (a < fc.A) {
        cr = fmaf(probs[a], pal[3 * a + 0], cr);
        cg = fmaf(probs[a], pal[3 * a + 1], cg);
        cb = fmaf(probs[a], pal[3 * a + 2], cb);
      }
    }
  } else {
    cr = sigmoid_fast(out[1]) * 2.004f - 1.002f;
    cg = sigmoid_fast(out[2]) * 2.004f - 1.002f;
    cb = sigmoid_fast(out[3]) * 2.004f - 1.002f;
  }
}

}  // namespace nfi
