// SDF point evaluator for the generator's regulariser heads (C ABI: include/nfi_heads.h;
// /root/reference/models/generator.py:520-585, lib/ops.py:58-120; SURVEY.md section 8f, N2).
//
//   forward   d(x)  = b2_0 + sum_j W2_0j softplus(pre_j),   pre_j = b1_j + sum_c W1_jc F_c(x)
//             g_k(x) = dd/dx_k = gamma sum_c t_c G_kc,       t_c = sum_j W1_jc v_j,  v_j = W2_0j sigmoid(pre_j)
//             F = mean over the three planes of the bilinear fetch, G_k = dF/d(texel coordinate k)
//             (gather_features_grad), gamma = (R-1)/2 / 3 / scene_range.  G follows the heads'
//             reference fetch (lib/ops.py grid_sample2d), not F.grid_sample: it is nonzero on the
//             lower faces (texel coordinate 0) and zero on the upper ones (make_taps<true>)
//   backward  of BOTH outputs (the eikonal loss differentiates g: a double backward in the
//             reference), with ghat = gamma * dL/dg:
//               tbar_c = sum_k ghat_k G_kc            vbar_j = sum_c W1_jc tbar_c
//               dL/dpre_j = vbar_j W2_0j s_j (1 - s_j) + dL/dd W2_0j s_j
//               dL/dF_c = sum_j W1_jc dL/dpre_j       dL/dG_kc = ghat_k t_c
//               dL/dW1_jc = dL/dpre_j F_c + v_j tbar_c    dL/db1_j = dL/dpre_j
//               dL/dW2_0j = vbar_j s_j + dL/dd a_j        dL/db2_0 = dL/dd
//             and the plane gradient scatters dL/dF with the bilinear weights and dL/dG with the
//             derivatives of the bilinear weights (red.global.add.v4, 8 lanes per texel).
// One thread = one point, a warp fetches / scatters its 32 points cooperatively; fp32 FFMA built
// from the device functions of the SIMT render kernels (nfi_common.cuh).  29,791 points per image
// against the render's 2.1 M: this is not a hot loop, it exists so that the GAN generator step
// does not need the unfused decoder (and its autograd graph) at all.
#include <cuda_runtime.h>

#include "nfi_common.cuh"
#include "nfi_heads.h"

namespace nfi {
namespace heads {

constexpr int kPRow = 68;  // padded 64-float row

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b),
               "f"(c), "f"(d)
               : "memory");
}

struct Smem {
  float* W1t;  // [32][64]  W1t[c*64 + j] = W1[j][c]
  float* b1;   // [64]
  float* w2r;  // [64]      row 0 of W2
  float* F;    // per warp [32][kFRow]
  float* G;    // per warp [3][32][kFRow]
  float* T;    // per warp [32][kFRow]      (backward)
  float* P;    // per warp [32][kPRow]      (backward)
  float* V;    // per warp [32][kPRow]      (backward)
};

__host__ __device__ inline size_t smem_floats(bool bwd) {
  size_t n = kC * kHid + kHid + kHid + kWarps * 32 * kFRow + kWarps * 3 * 32 * kFRow;
  if (bwd) n += kWarps * 32 * kFRow + 2 * kWarps * 32 * kPRow;
  return n;
}

__device__ __forceinline__ Smem carve(float* q, bool bwd) {
  Smem s;
  s.W1t = q; q += kC * kHid;
  s.b1 = q; q += kHid;
  s.w2r = q; q += kHid;
  s.F = q; q += kWarps * 32 * kFRow;
  s.G = q; q += kWarps * 3 * 32 * kFRow;
  s.T = s.P = s.V = nullptr;
  if (bwd) {
    s.T = q; q += kWarps * 32 * kFRow;
    s.P = q; q += kWarps * 32 * kPRow;
    s.V = q;
  }
  return s;
}

__device__ __forceinline__ void load_weights(const nfi_sdf_points_params& p, const Smem& s, int tid) {
  for (int i = tid; i < kC * kHid; i += kThreads) {
    const int c = i / kHid, j = i % kHid;
    s.W1t[i] = p.w1[j * kC + c];
  }
  for (int i = tid; i < kHid; i += kThreads) {
    s.b1[i] = p.b1[i];
    s.w2r[i] = p.w2[i];
  }
}

// pre-activations of this lane's point from its feature row
__device__ __forceinline__ void pre_activations(const float* __restrict__ frow, const Smem& s,
                                                float (&h)[kHid]) {
#pragma unroll
  for (int j4 = 0; j4 < kHid / 4; ++j4) {
    const float4 bv = *reinterpret_cast<const float4*>(s.b1 + 4 * j4);
    h[4 * j4 + 0] = bv.x; h[4 * j4 + 1] = bv.y; h[4 * j4 + 2] = bv.z; h[4 * j4 + 3] = bv.w;
  }
#pragma unroll 1
  for (int c = 0; c < kC; ++c) {
    const float f = frow[c];
    const float4* wr = reinterpret_cast<const float4*>(s.W1t + c * kHid);
#pragma unroll
    for (int j4 = 0; j4 < kHid / 4; ++j4) {
      const float4 w = wr[j4];
      h[4 * j4 + 0] = fmaf(w.x, f, h[4 * j4 + 0]);
      h[4 * j4 + 1] = fmaf(w.y, f, h[4 * j4 + 1]);
      h[4 * j4 + 2] = fmaf(w.z, f, h[4 * j4 + 2]);
      h[4 * j4 + 3] = fmaf(w.w, f, h[4 * j4 + 3]);
    }
  }
}

// sum_j W1t[c][j] * v[j]
__device__ __forceinline__ float dot_w1_row(const Smem& s, int c, const float (&v)[kHid]) {
  const float4* wr = reinterpret_cast<const float4*>(s.W1t + c * kHid);
  float u = 0.f;
#pragma unroll
  for (int j4 = 0; j4 < kHid / 4; ++j4) {
    const float4 w = wr[j4];
    u = fmaf(w.x, v[4 * j4 + 0], u);
    u = fmaf(w.y, v[4 * j4 + 1], u);
    u = fmaf(w.z, v[4 * j4 + 2], u);
    u = fmaf(w.w, v[4 * j4 + 3], u);
  }
  return u;
}

__device__ __forceinline__ float sigmoid_sp(float x) {  // d softplus(x, threshold 20) / dx
  return x > 20.f ? 1.f : 1.f / (1.f + expf(-x));
}
__device__ __forceinline__ float softplus_sp(float x) {
  return x > 20.f ? x : fmaxf(x, 0.f) + log1pf(expf(-fabsf(x)));
}

struct Unit {
  int b;
  long long row;  // b * N + idx (clamped)
  bool valid;
  float x0, x1, x2;
};
__device__ __forceinline__ Unit load_unit(const nfi_sdf_points_params& p, long long u, long long nb,
                                          int lane) {
  Unit q;
  q.b = (int)(u / nb);
  const long long idx = (u % nb) * 32 + lane;
  q.valid = idx < p.n_points;
  q.row = (long long)q.b * p.n_points + (q.valid ? idx : p.n_points - 1);
  q.x0 = p.points[q.row * 3 + 0] / p.scene_range;
  q.x1 = p.points[q.row * 3 + 1] / p.scene_range;
  q.x2 = p.points[q.row * 3 + 2] / p.scene_range;
  return q;
}

__global__ void __launch_bounds__(kThreads)
sdf_points_fwd_kernel(const nfi_sdf_points_params p) {
  extern __shared__ __align__(16) float smem_f[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const Smem s = carve(smem_f, false);
  load_weights(p, s, tid);
  __syncthreads();
  const float b2_0 = p.b2[0];
  const float gamma = 0.5f * (float)(p.plane_res - 1) / (3.f * p.scene_range);
  float* Fw = s.F + warp * 32 * kFRow;
  float* Gw = s.G + warp * 3 * 32 * kFRow;
  const long long nb = (p.n_points + 31) / 32, units = nb * p.batch;
  const size_t plane_img = (size_t)3 * p.plane_res * p.plane_res * kC;
  for (long long u = (long long)blockIdx.x * kWarps + warp; u < units; u += (long long)gridDim.x * kWarps) {
    const Unit q = load_unit(p, u, nb, lane);
    gather_features_grad<true>(p.planes + q.b * plane_img, p.plane_res, q.x0, q.x1, q.x2, Fw, Gw,
                               lane);
    float h[kHid];
    pre_activations(Fw + lane * kFRow, s, h);
    float d = b2_0;
#pragma unroll
    for (int j = 0; j < kHid; ++j) {
      d = fmaf(s.w2r[j], softplus_sp(h[j]), d);
      h[j] = s.w2r[j] * sigmoid_sp(h[j]);  // v_j
    }
    if (q.valid) p.d[q.row] = d;
    if (p.grad != nullptr) {
      float g0 = 0.f, g1 = 0.f, g2 = 0.f;
#pragma unroll 1
      for (int c = 0; c < kC; ++c) {
        const float t = dot_w1_row(s, c, h);
        g0 = fmaf(t, Gw[lane * kFRow + c], g0);
        g1 = fmaf(t, Gw[(32 + lane) * kFRow + c], g1);
        g2 = fmaf(t, Gw[(64 + lane) * kFRow + c], g2);
      }
      if (q.valid) {
        p.grad[q.row * 3 + 0] = g0 * gamma;
        p.grad[q.row * 3 + 1] = g1 * gamma;
        p.grad[q.row * 3 + 2] = g2 * gamma;
      }
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(kThreads)
sdf_points_bwd_kernel(const nfi_sdf_points_params p, const nfi_sdf_points_grads g) {
  extern __shared__ __align__(16) float smem_f[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const Smem s = carve(smem_f, true);
  load_weights(p, s, tid);
  __syncthreads();
  const float gamma = 0.5f * (float)(p.plane_res - 1) / (3.f * p.scene_range);
  float* Fw = s.F + warp * 32 * kFRow;
  float* Gw = s.G + warp * 3 * 32 * kFRow;
  float* Tw = s.T + warp * 32 * kFRow;
  float* Pw = s.P + warp * 32 * kPRow;
  float* Vw = s.V + warp * 32 * kPRow;
  const bool wgrad = g.grad_w1 != nullptr;
  const int j0 = 2 * lane;  // this lane accumulates rows j0, j0 + 1 of dW1 / db1 / dW2_0
  float acc_w1[2 * kC];
  float acc_b1[2] = {0.f, 0.f}, acc_w2[2] = {0.f, 0.f}, acc_b2 = 0.f;
#pragma unroll
  for (int i = 0; i < 2 * kC; ++i) acc_w1[i] = 0.f;
  const long long nb = (p.n_points + 31) / 32, units = nb * p.batch;
  const size_t plane_img = (size_t)3 * p.plane_res * p.plane_res * kC;
  const size_t plane_stride = (size_t)p.plane_res * p.plane_res * kC;
  for (long long u = (long long)blockIdx.x * kWarps + warp; u < units; u += (long long)gridDim.x * kWarps) {
    const Unit q = load_unit(p, u, nb, lane);
    const float gd = (q.valid && g.g_d) ? g.g_d[q.row] : 0.f;
    float gh0 = 0.f, gh1 = 0.f, gh2 = 0.f;
    if (q.valid && g.g_grad) {
      gh0 = gamma * g.g_grad[q.row * 3 + 0];
      gh1 = gamma * g.g_grad[q.row * 3 + 1];
      gh2 = gamma * g.g_grad[q.row * 3 + 2];
    }
    const float* planes_b = p.planes + q.b * plane_img;
    gather_features_grad<true>(planes_b, p.plane_res, q.x0, q.x1, q.x2, Fw, Gw, lane);
    float h[kHid], vb[kHid];
    pre_activations(Fw + lane * kFRow, s, h);
    // tbar_c -> Tw row; vbar_j = sum_c W1_jc tbar_c
#pragma unroll
    for (int j = 0; j < kHid; ++j) vb[j] = 0.f;
#pragma unroll 1
    for (int c = 0; c < kC; ++c) {
      const float tb = gh0 * Gw[lane * kFRow + c] + gh1 * Gw[(32 + lane) * kFRow + c] +
                       gh2 * Gw[(64 + lane) * kFRow + c];
      Tw[lane * kFRow + c] = tb;
      const float4* wr = reinterpret_cast<const float4*>(s.W1t + c * kHid);
#pragma unroll
      for (int j4 = 0; j4 < kHid / 4; ++j4) {
        const float4 w = wr[j4];
        vb[4 * j4 + 0] = fmaf(w.x, tb, vb[4 * j4 + 0]);
        vb[4 * j4 + 1] = fmaf(w.y, tb, vb[4 * j4 + 1]);
        vb[4 * j4 + 2] = fmaf(w.z, tb, vb[4 * j4 + 2]);
        vb[4 * j4 + 3] = fmaf(w.w, tb, vb[4 * j4 + 3]);
      }
    }
    // per hidden unit: h <- dL/dpre, vb <- q (the dW2_0 term), Vw row <- v, Pw row <- dL/dpre
#pragma unroll
    for (int j = 0; j < kHid; ++j) {
      const float sj = sigmoid_sp(h[j]), aj = softplus_sp(h[j]), w2 = s.w2r[j];
      const float pbar = vb[j] * w2 * (sj * (1.f - sj)) + gd * w2 * sj;
      Vw[lane * kPRow + j] = w2 * sj;
      Pw[lane * kPRow + j] = pbar;
      vb[j] = vb[j] * sj + gd * aj;
      h[j] = pbar;
    }
    acc_b2 += gd;
    __syncwarp();
    if (wgrad) {
      // dW1[j][c] += pbar[pt][j] F[pt][c] + v[pt][j] tbar[pt][c]   (rows j0, j0 + 1)
#pragma unroll 1
      for (int pt = 0; pt < 32; ++pt) {
        const float2 pj = *reinterpret_cast<const float2*>(Pw + pt * kPRow + j0);
        const float2 vj = *reinterpret_cast<const float2*>(Vw + pt * kPRow + j0);
        acc_b1[0] += pj.x;
        acc_b1[1] += pj.y;
#pragma unroll
        for (int c4 = 0; c4 < kC / 4; ++c4) {
          const float4 f4 = *reinterpret_cast<const float4*>(Fw + pt * kFRow + 4 * c4);
          const float4 t4 = *reinterpret_cast<const float4*>(Tw + pt * kFRow + 4 * c4);
          const float fv[4] = {f4.x, f4.y, f4.z, f4.w}, tv[4] = {t4.x, t4.y, t4.z, t4.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            acc_w1[4 * c4 + e] = fmaf(pj.x, fv[e], fmaf(vj.x, tv[e], acc_w1[4 * c4 + e]));
            acc_w1[kC + 4 * c4 + e] = fmaf(pj.y, fv[e], fmaf(vj.y, tv[e], acc_w1[kC + 4 * c4 + e]));
          }
        }
      }
      __syncwarp();
    }
    // own row: dL/dF_c (-> Fw) and t_c (-> Tw); v is read back from this lane's Vw row
    {
      float v[kHid];
#pragma unroll
      for (int j4 = 0; j4 < kHid / 4; ++j4) {
        const float4 t = *reinterpret_cast<const float4*>(Vw + lane * kPRow + 4 * j4);
        v[4 * j4 + 0] = t.x; v[4 * j4 + 1] = t.y; v[4 * j4 + 2] = t.z; v[4 * j4 + 3] = t.w;
      }
#pragma unroll 1
      for (int c = 0; c < kC; ++c) {
        Fw[lane * kFRow + c] = dot_w1_row(s, c, h) * (1.f / 3.f);  // per-plane share of the mean
        Tw[lane * kFRow + c] = dot_w1_row(s, c, v);
      }
    }
    if (wgrad) {
      __syncwarp();
#pragma unroll
      for (int j = 0; j < kHid; ++j) Vw[lane * kPRow + j] = vb[j];
      __syncwarp();
#pragma unroll 1
      for (int pt = 0; pt < 32; ++pt) {
        const float2 qj = *reinterpret_cast<const float2*>(Vw + pt * kPRow + j0);
        acc_w2[0] += qj.x;
        acc_w2[1] += qj.y;
      }
    }
    __syncwarp();
    // scatter: 8 lanes per texel, 4 points per iteration
    if (g.grad_planes != nullptr) {
      float* gplanes_b = g.grad_planes + q.b * plane_img;
      const int qq = lane >> 3, kq = lane & 7;
#pragma unroll 1
      for (int gi = 0; gi < 8; ++gi) {
        const int src = 4 * gi + qq;
        const float c0 = __shfl_sync(kFull, q.x0, src), c1 = __shfl_sync(kFull, q.x1, src),
                    c2 = __shfl_sync(kFull, q.x2, src);
        const float a0 = __shfl_sync(kFull, gh0, src), a1 = __shfl_sync(kFull, gh1, src),
                    a2 = __shfl_sync(kFull, gh2, src);
        const bool ok = __shfl_sync(kFull, (int)q.valid, src) != 0;
        const float4 f4 = *reinterpret_cast<const float4*>(Fw + src * kFRow + 4 * kq);
        const float4 t4 = *reinterpret_cast<const float4*>(Tw + src * kFRow + 4 * kq);
        if (!ok) continue;
#pragma unroll
        for (int pl = 0; pl < 3; ++pl) {
          const float ga = (pl == 2) ? c1 : c0, gb = (pl == 0) ? c1 : c2;
          const float ha = (pl == 2) ? a1 : a0, hb = (pl == 0) ? a1 : a2;  // ghat of the two axes
          const Taps t = make_taps<true>(ga, gb, p.plane_res);
          const float A = t.inx ? ha : 0.f, Bc = t.iny ? hb : 0.f;
          float* gp = gplanes_b + pl * plane_stride + 4 * kq;
          const float k00 = -t.gy0 * A - t.gx0 * Bc, k01 = t.gy0 * A - t.gx1 * Bc,
                      k10 = -t.gy1 * A + t.gx0 * Bc, k11 = t.gy1 * A + t.gx1 * Bc;
          red_add_v4(gp + (size_t)t.o00 * kC, fmaf(f4.x, t.w00, t4.x * k00), fmaf(f4.y, t.w00, t4.y * k00),
                     fmaf(f4.z, t.w00, t4.z * k00), fmaf(f4.w, t.w00, t4.w * k00));
          red_add_v4(gp + (size_t)t.o01 * kC, fmaf(f4.x, t.w01, t4.x * k01), fmaf(f4.y, t.w01, t4.y * k01),
                     fmaf(f4.z, t.w01, t4.z * k01), fmaf(f4.w, t.w01, t4.w * k01));
          red_add_v4(gp + (size_t)t.o10 * kC, fmaf(f4.x, t.w10, t4.x * k10), fmaf(f4.y, t.w10, t4.y * k10),
                     fmaf(f4.z, t.w10, t4.z * k10), fmaf(f4.w, t.w10, t4.w * k10));
          red_add_v4(gp + (size_t)t.o11 * kC, fmaf(f4.x, t.w11, t4.x * k11), fmaf(f4.y, t.w11, t4.y * k11),
                     fmaf(f4.z, t.w11, t4.z * k11), fmaf(f4.w, t.w11, t4.w * k11));
        }
      }
    }
    __syncwarp();
  }
  if (wgrad) {
#pragma unroll
    for (int c = 0; c < kC; ++c) {
      atomicAdd(g.grad_w1 + (size_t)j0 * kC + c, acc_w1[c]);
      atomicAdd(g.grad_w1 + (size_t)(j0 + 1) * kC + c, acc_w1[kC + c]);
    }
    if (g.grad_b1) {
      atomicAdd(g.grad_b1 + j0, acc_b1[0]);
      atomicAdd(g.grad_b1 + j0 + 1, acc_b1[1]);
    }
    if (g.grad_w2_row0) {
      atomicAdd(g.grad_w2_row0 + j0, acc_w2[0]);
      atomicAdd(g.grad_w2_row0 + j0 + 1, acc_w2[1]);
    }
    if (g.grad_b2_0) {
      const float sb = warp_sum(acc_b2);
      if (lane == 0) atomicAdd(g.grad_b2_0, sb);
    }
  }
}

static unsigned grid_for(const nfi_sdf_points_params& p) {
  const long long units = ((p.n_points + 31) / 32) * p.batch;
  long long ctas = (units + kWarps - 1) / kWarps;
  if (ctas > 148 * 4) ctas = 148 * 4;  // persistent: the backward keeps dW accumulators per lane
  return (unsigned)(ctas < 1 ? 1 : ctas);
}

int launch_forward(const nfi_sdf_points_params& p, cudaStream_t st) {
  const size_t smem = smem_floats(false) * sizeof(float);
  NFI_CUDA(cudaFuncSetAttribute(sdf_points_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)smem));
  sdf_points_fwd_kernel<<<grid_for(p), kThreads, smem, st>>>(p);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int launch_backward(const nfi_sdf_points_params& p, const nfi_sdf_points_grads& g,
                    cudaStream_t st) {
  const size_t smem = smem_floats(true) * sizeof(float);
  NFI_CUDA(cudaFuncSetAttribute(sdf_points_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)smem));
  sdf_points_bwd_kernel<<<grid_for(p), kThreads, smem, st>>>(p, g);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace heads
}  // namespace nfi

using nfi::fail;

extern "C" {

static int check_sdf_points(const nfi_sdf_points_params* p) {
  if (p == nullptr) return fail("params is NULL");
  if (p->batch <= 0 || p->n_points <= 0 || p->plane_res < 2) return fail("empty batch / no points");
  if (!p->planes || !p->w1 || !p->b1 || !p->w2 || !p->b2 || !p->points)
    return fail("planes, decoder weights and points must be given");
  if (!(p->scene_range > 0.f)) return fail("scene_range must be positive");
  return 0;
}

int nfi_sdf_points_forward(const nfi_sdf_points_params* params, void* stream) {
  if (const int rc = check_sdf_points(params)) return rc;
  if (!params->d) return fail("output d must be given");
  return nfi::heads::launch_forward(*params, (cudaStream_t)stream);
}

int nfi_sdf_points_backward(const nfi_sdf_points_params* params, const nfi_sdf_points_grads* grads,
                            void* stream) {
  if (const int rc = check_sdf_points(params)) return rc;
  if (grads == nullptr) return fail("grads is NULL");
  if (!grads->g_d && !grads->g_grad) return fail("no upstream gradient");
  if (grads->grad_w1 && (!grads->grad_b1 || !grads->grad_w2_row0 || !grads->grad_b2_0))
    return fail("decoder gradients come as a set: grad_w1, grad_b1, grad_w2_row0, grad_b2_0");
  return nfi::heads::launch_backward(*params, *grads, (cudaStream_t)stream);
}

}  // extern "C"
