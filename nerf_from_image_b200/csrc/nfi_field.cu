// Translation unit of the two small neighbours of the render path:
//   * sample_field_simt   -- the generator's `sampler` closure at arbitrary points
//                            (models/generator.py:587-681; SURVEY.md section 8b, seam B2)
//   * pose_to_matrix_*    -- lib/pose_utils.py:32-70 and its vector-Jacobian product
//                            (SURVEY.md section 8f, N4)
// fp32 SIMT arithmetic built from the same device functions as render_forward_simt
// (nfi_common.cuh), so a point evaluated here and the same point evaluated along a ray agree.
#include <cuda_runtime.h>
#include <string.h>

#include "nfi_common.cuh"
#include "nfi_render.h"
#include "nfi_forward.cuh"

namespace nfi {
namespace {

// One thread = one point; a warp fetches its 32 points' features cooperatively.  blockIdx.y is
// the image, blockIdx.x the 128-point chunk.  `p` carries the field (planes, decoder, palette,
// beta/alpha, scene_range): the same struct the render kernels read, so load_weights_smem and
// field_head are shared.
template <int NOUT_PAD, bool NORM>
__global__ void __launch_bounds__(kThreads)
sample_field_simt(const nfi_render_params p, const nfi_sample_params io) {
  extern __shared__ __align__(16) float smem_f[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  FwdSmem sm;
  {
    float* q = smem_f;
    sm.W1t = q; q += kC * kHid;
    sm.b1 = q; q += kHid;
    sm.W2t = q; q += kHid * NOUT_PAD;
    sm.b2 = q; q += NOUT_PAD;
    sm.pal = q; q += 48;
    sm.F = q; q += kWarps * 32 * kFRow;
    sm.G = q;
    sm.colA = sm.colB = nullptr;
    sm.W3t = sm.b3 = sm.xs = nullptr;
  }
  const int b = blockIdx.y;
  load_weights_smem<NOUT_PAD>(p, b, sm, tid, 1 + (p.n_attention > 0 ? p.n_attention : 3));
  __syncthreads();

  const long long n = io.n_points;
  const long long idx = (long long)blockIdx.x * kThreads + tid;
  const bool valid = idx < n;
  const long long row = (long long)b * n + (valid ? idx : n - 1);  // idle lanes redo the last point

  const float wx = io.points[row * 3 + 0], wy = io.points[row * 3 + 1], wz = io.points[row * 3 + 2];
  const float x0 = wx / p.scene_range, x1 = wy / p.scene_range, x2 = wz / p.scene_range;
  const float keep = (fabsf(x0) > 1.f || fabsf(x1) > 1.f || fabsf(x2) > 1.f) ? 0.f : 1.f;

  FieldConst fc;
  fc.A = p.n_attention;
  fc.use_sdf = p.use_sdf;
  fc.inv_beta = p.use_sdf ? 1.f / p.beta[0] : 0.f;
  fc.inv_alpha = p.use_sdf ? 1.f / p.alpha[0] : 0.f;

  const float* planes_b = p.planes + (size_t)b * 3 * p.plane_res * p.plane_res * kC;
  float* Fw = sm.F + warp * 32 * kFRow;
  const float* frow = Fw + lane * kFRow;
  float out[NOUT_PAD];
  float h[kHid];
  float n0 = 0.f, n1 = 0.f, n2 = 0.f;
  if (NORM) {
    float* Gw = sm.G + warp * 3 * 32 * kFRow;
    gather_features_grad(planes_b, p.plane_res, x0, x1, x2, Fw, Gw, lane);
    mlp_forward<NOUT_PAD, true>(frow, sm.W1t, sm.b1, sm.W2t, sm.b2, out, h);
    sdf_gradient<NOUT_PAD>(h, sm.W1t, sm.W2t, Gw, lane, n0, n1, n2);
    const float sc = 0.5f * (float)(p.plane_res - 1) / (3.f * p.scene_range);
    n0 *= sc;
    n1 *= sc;
    n2 *= sc;
    const float inv = 1.f / fmaxf(sqrtf((n0 * n0 + n1 * n1) + n2 * n2), 1e-12f);  // F.normalize
    n0 *= inv;
    n1 *= inv;
    n2 *= inv;
  } else {
    gather_features(planes_b, p.plane_res, x0, x1, x2, Fw, lane);
    mlp_forward<NOUT_PAD, false>(frow, sm.W1t, sm.b1, sm.W2t, sm.b2, out, h);
  }
  float sigma, cr, cg, cb;
  float probs[NOUT_PAD];
  field_head<NOUT_PAD>(out, fc, sm.pal, keep, sigma, cr, cg, cb, probs);
  if (io.bbox_debug) {
    // generator.py:640-657: +100 where, for every pair of axes, at least one coordinate is
    // within eps of the cube face (the twelve edges), inside the cube only
    const float lim = p.scene_range - 5e-2f;
    const bool ix = fabsf(wx) < lim, iy = fabsf(wy) < lim, iz = fabsf(wz) < lim;
    const float edge = ((ix && iy) || (ix && iz) || (iy && iz)) ? 0.f : 1.f;
    sigma += 100.f * (edge * keep);
  }
  if (!valid) return;
  if (io.sdf_distance) io.sdf_distance[row] = out[0];
  if (io.sigma) io.sigma[row] = sigma;
  if (io.rgb) {
    io.rgb[row * 3 + 0] = cr;
    io.rgb[row * 3 + 1] = cg;
    io.rgb[row * 3 + 2] = cb;
  }
  if (io.semantics && p.n_attention > 0) {
#pragma unroll
    for (int a = 0; a < NOUT_PAD - 1; ++a)
      if (a < p.n_attention) io.semantics[row * p.n_attention + a] = probs[a];
  }
  if (NORM && io.normals) {
    io.normals[row * 3 + 0] = n0;
    io.normals[row * 3 + 1] = n1;
    io.normals[row * 3 + 2] = n2;
  }
}

template <int NP, bool NORM>
int run_sampler(const nfi_render_params& p, const nfi_sample_params& io, cudaStream_t st) {
  const size_t smem = fwd_smem_floats(NP, 0, false, NORM) * sizeof(float);
  auto k = sample_field_simt<NP, NORM>;
  NFI_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid((unsigned)((io.n_points + kThreads - 1) / kThreads), (unsigned)io.batch);
  k<<<grid, kThreads, smem, st>>>(p, io);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------ pose_to_matrix
// quaternion_rotate_vector(q, e_i) for the three unit vectors (lib/pose_utils.py:32-44):
// R[i] = e_i + 2 (w (qv x e_i) + qv x (qv x e_i)), written with the cross products of the
// reference so the rounding follows it.
__device__ __forceinline__ void cross3(const float* a, const float* b, float* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

__device__ __forceinline__ void quat_rows(const float* q, float (&R)[3][3]) {
  const float qv[3] = {q[1], q[2], q[3]};
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float e[3] = {0.f, 0.f, 0.f};
    e[i] = 1.f;
    float uv[3], uuv[3];
    cross3(qv, e, uv);
    cross3(qv, uv, uuv);
#pragma unroll
    for (int c = 0; c < 3; ++c) R[i][c] = e[c] + 2.f * (q[0] * uv[c] + uuv[c]);
  }
}

__global__ void pose_to_matrix_kernel(const float* __restrict__ z0, const float* __restrict__ t2,
                                      const float* __restrict__ s, const float* __restrict__ q,
                                      int flipped, int batch, float* __restrict__ c2w,
                                      float* __restrict__ focal) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  float R[3][3];
  quat_rows(q + 4 * b, R);
  const float sb = s[b];
  float t3[3];
  float f = 0.f;
  if (z0 != nullptr) {
    f = 1.f + expf(z0[b]);
    t3[0] = t2[2 * b + 0] / sb;
    t3[1] = t2[2 * b + 1] / sb;
    t3[2] = f / sb;
  } else {
    t3[0] = t2[2 * b + 0];
    t3[1] = t2[2 * b + 1];
    t3[2] = 10.f;
  }
  float M[16];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int c = 0; c < 3; ++c) M[4 * i + c] = R[i][c];
    M[4 * i + 3] = (t3[0] * R[i][0] + t3[1] * R[i][1]) + t3[2] * R[i][2];
  }
  M[12] = M[13] = M[14] = 0.f;
  M[15] = 1.f;
  if (flipped) {
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      M[4 * i + 1] *= -1.f;
      M[4 * i + 2] *= -1.f;
      M[4 * i + 3] *= -1.f;
    }
  }
  if (z0 == nullptr) {
#pragma unroll
    for (int i = 0; i < 16; ++i) M[i] = M[i] / sb;
  } else if (focal != nullptr) {
    focal[b] = f / 2.f;
  }
#pragma unroll
  for (int i = 0; i < 16; ++i) c2w[16 * b + i] = M[i];
}

__global__ void pose_to_matrix_bwd_kernel(const float* __restrict__ z0,
                                          const float* __restrict__ t2,
                                          const float* __restrict__ s, const float* __restrict__ q,
                                          int flipped, int batch, const float* __restrict__ g_c2w,
                                          const float* __restrict__ g_focal,
                                          float* __restrict__ g_z0, float* __restrict__ g_t2,
                                          float* __restrict__ g_s, float* __restrict__ g_q) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  float R[3][3];
  quat_rows(q + 4 * b, R);
  const float sb = s[b];
  const bool persp = z0 != nullptr;
  float t3[3];
  float f = 0.f;
  if (persp) {
    f = 1.f + expf(z0[b]);
    t3[0] = t2[2 * b + 0] / sb;
    t3[1] = t2[2 * b + 1] / sb;
    t3[2] = f / sb;
  } else {
    t3[0] = t2[2 * b + 0];
    t3[1] = t2[2 * b + 1];
    t3[2] = 10.f;
  }
  // upstream gradient of the un-flipped, un-scaled 3x4 block
  float G[3][4];
  float gs = 0.f;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float g = g_c2w[16 * b + 4 * i + c];
      if (!persp) {
        // out = inner / s:  d inner = g / s,  ds -= g * inner / s^2
        float inner = (c < 3) ? R[i][c] : (t3[0] * R[i][0] + t3[1] * R[i][1]) + t3[2] * R[i][2];
        if (flipped && c > 0) inner = -inner;
        gs -= g * inner / (sb * sb);
        g = g / sb;
      }
      if (flipped && c > 0) g = -g;
      G[i][c] = g;
    }
  if (!persp) gs -= g_c2w[16 * b + 15] / (sb * sb);  // element [3,3] = 1 / s
  // translation = R t3
  float gR[3][3];
  float gt3[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      gR[i][c] = G[i][c] + G[i][3] * t3[c];
      gt3[c] += G[i][3] * R[i][c];
    }
  if (persp) {
    g_t2[2 * b + 0] = gt3[0] / sb;
    g_t2[2 * b + 1] = gt3[1] / sb;
    gs -= ((gt3[0] * t3[0] + gt3[1] * t3[1]) + gt3[2] * t3[2]) / sb;
    float gf = gt3[2] / sb;
    if (g_focal != nullptr) gf += 0.5f * g_focal[b];
    g_z0[b] = gf * (f - 1.f);
  } else {
    g_t2[2 * b + 0] = gt3[0];
    g_t2[2 * b + 1] = gt3[1];
  }
  g_s[b] = gs;
  // rows R_i = e_i + 2 w (qv x e_i) + 2 (qv (qv.e_i) - e_i (qv.qv))
  const float w = q[4 * b + 0];
  const float qv[3] = {q[4 * b + 1], q[4 * b + 2], q[4 * b + 3]};
  float gw = 0.f;
  float gq[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float e[3] = {0.f, 0.f, 0.f};
    e[i] = 1.f;
    const float* g = gR[i];
    float uv[3], exg[3];
    cross3(qv, e, uv);
    cross3(e, g, exg);
    gw += 2.f * ((g[0] * uv[0] + g[1] * uv[1]) + g[2] * uv[2]);
    const float gdq = (g[0] * qv[0] + g[1] * qv[1]) + g[2] * qv[2];
    const float qde = qv[i], gde = g[i];
#pragma unroll
    for (int c = 0; c < 3; ++c)
      gq[c] += 2.f * w * exg[c] + 2.f * (g[c] * qde + e[c] * gdq - 2.f * gde * qv[c]);
  }
  g_q[4 * b + 0] = gw;
  g_q[4 * b + 1] = gq[0];
  g_q[4 * b + 2] = gq[1];
  g_q[4 * b + 3] = gq[2];
}

}  // namespace

int launch_sample_field(const nfi_render_params& p, const nfi_sample_params& io, int nout_pad,
                        cudaStream_t st) {
  const bool norm = io.normals != nullptr;
  switch (nout_pad) {
    case 4:
      return norm ? run_sampler<4, true>(p, io, st) : run_sampler<4, false>(p, io, st);
    case 12:
      return norm ? run_sampler<12, true>(p, io, st) : run_sampler<12, false>(p, io, st);
    default:
      return norm ? run_sampler<16, true>(p, io, st) : run_sampler<16, false>(p, io, st);
  }
}

int launch_pose_to_matrix(const float* z0, const float* t2, const float* s, const float* q,
                          int flipped, int batch, float* c2w, float* focal, cudaStream_t st) {
  pose_to_matrix_kernel<<<(batch + 63) / 64, 64, 0, st>>>(z0, t2, s, q, flipped, batch, c2w,
                                                          focal);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int launch_pose_to_matrix_backward(const float* z0, const float* t2, const float* s,
                                   const float* q, int flipped, int batch, const float* g_c2w,
                                   const float* g_focal, float* g_z0, float* g_t2, float* g_s,
                                   float* g_q, cudaStream_t st) {
  pose_to_matrix_bwd_kernel<<<(batch + 63) / 64, 64, 0, st>>>(z0, t2, s, q, flipped, batch, g_c2w,
                                                              g_focal, g_z0, g_t2, g_s, g_q);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace nfi

using nfi::fail;

extern "C" {

int nfi_sample_field(const nfi_sample_params* sp, void* stream) {
  if (sp == nullptr) return fail("params is NULL");
  if (sp->batch <= 0 || sp->batch > 65535 || sp->n_points <= 0) return fail("empty point set");
  if (sp->n_points > ((int64_t)1 << 37)) return fail("too many points per image");
  if (sp->plane_res < 2) return fail("plane_res must be >= 2");
  if (sp->n_attention < 0 || sp->n_attention > NFI_MAX_ATTENTION)
    return fail("attention_values must be in [0, 15]");
  if (!(sp->scene_range > 0.f)) return fail("scene_range must be positive");
  if (!sp->planes || !sp->w1 || !sp->b1 || !sp->w2 || !sp->b2 || !sp->points)
    return fail("planes / decoder weights / points must be given");
  if (sp->n_attention > 0 && !sp->palette)
    return fail("palette missing (attention_values > 0)");
  if (sp->use_sdf && (!sp->beta || !sp->alpha)) return fail("use_sdf needs beta and alpha");
  if (sp->semantics && sp->n_attention <= 0)
    return fail("'semantics' needs attention_values > 0");  // generator.py:673
  if (sp->normals && !sp->use_sdf) return fail("'normals' needs use_sdf");  // generator.py:600
  if (sp->bbox_debug && !sp->sigma) return fail("bbox_debug modifies sigma: request it");
  if (!sp->sdf_distance && !sp->sigma && !sp->rgb && !sp->semantics && !sp->normals)
    return fail("no sampler output requested");
  nfi_render_params p;
  memset(&p, 0, sizeof(p));
  p.batch = sp->batch;
  p.plane_res = sp->plane_res;
  p.n_attention = sp->n_attention;
  p.use_sdf = sp->use_sdf;
  p.scene_range = sp->scene_range;
  p.planes = sp->planes;
  p.w1 = sp->w1;
  p.b1 = sp->b1;
  p.w2 = sp->w2;
  p.b2 = sp->b2;
  p.palette = sp->palette;
  p.beta = sp->beta;
  p.alpha = sp->alpha;
  return nfi::launch_sample_field(p, *sp, nfi::nout_pad_of(p.n_attention), (cudaStream_t)stream);
}

int nfi_pose_to_matrix(const float* z0, const float* t2, const float* s, const float* q,
                       int32_t camera_flipped, int32_t batch, float* c2w, float* focal,
                       void* stream) {
  if (batch <= 0) return fail("empty batch");
  if (!t2 || !s || !q || !c2w) return fail("t2 / s / q / c2w must be given");
  if (z0 && !focal) return fail("perspective pose (z0 given) needs the focal output");
  return nfi::launch_pose_to_matrix(z0, t2, s, q, camera_flipped, batch, c2w, focal,
                                    (cudaStream_t)stream);
}

int nfi_pose_to_matrix_backward(const float* z0, const float* t2, const float* s, const float* q,
                                int32_t camera_flipped, int32_t batch, const float* g_c2w,
                                const float* g_focal, float* g_z0, float* g_t2, float* g_s,
                                float* g_q, void* stream) {
  if (batch <= 0) return fail("empty batch");
  if (!t2 || !s || !q || !g_c2w || !g_t2 || !g_s || !g_q)
    return fail("t2 / s / q / g_c2w and the three gradient outputs must be given");
  if (z0 && !g_z0) return fail("perspective pose (z0 given) needs g_z0");
  return nfi::launch_pose_to_matrix_backward(z0, t2, s, q, camera_flipped, batch, g_c2w, g_focal,
                                             g_z0, g_t2, g_s, g_q, (cudaStream_t)stream);
}

}  // extern "C"
