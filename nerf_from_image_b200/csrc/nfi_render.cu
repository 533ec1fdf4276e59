// C-ABI entry points of libnfi_render.so (see include/nfi_render.h).
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a --fmad=false -lineinfo
//        (nerf_from_image_b200/csrc/build.sh).  No torch, no CPU fallback: on a
//        machine without an sm_90 device every launch returns an error.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include "nfi_backward.cuh"
#include "nfi_forward.cuh"
#include "nfi_forward_tc.cuh"
#include "nfi_field_launch.h"
#include "nfi_pipe_launch.h"
#include "nfi_viewdir_launch.h"
#include "nfi_render.h"
#include "nfi_heads.h"
#include "nfi_heads_launch.h"
#include "nfi_synth.h"
#include "nfi_synth_launch.h"

#define NFI_STR_(x) #x
#define NFI_STR(x) NFI_STR_(x)

namespace {

thread_local char g_err[512] = "";

int fail(const char* fmt, const char* detail = "") {
  snprintf(g_err, sizeof(g_err), fmt, detail);
  return 1;
}

#define NFI_CUDA(expr)                                                      \
  do {                                                                      \
    cudaError_t e__ = (expr);                                               \
    if (e__ != cudaSuccess) {                                               \
      snprintf(g_err, sizeof(g_err), "%s failed: %s", #expr,                \
               cudaGetErrorString(e__));                                    \
      return 2;                                                             \
    }                                                                       \
  } while (0)

int nout_pad_of(const nfi_render_params* p) {
  const int nout = 1 + (p->n_attention > 0 ? p->n_attention : 3);
  return nout <= 4 ? 4 : (nout <= 12 ? 12 : 16);
}

int check_params(const nfi_render_params* p) {
  if (p == nullptr) return fail("params is NULL");
  if (p->batch <= 0 || p->height <= 0 || p->width <= 0) return fail("empty render");
  if (p->num_samples < 4 || p->num_samples > 512)
    return fail("depth_samples_per_ray must be in [4, 512]");
  if (p->plane_res < 2) return fail("plane_res must be >= 2");
  if (p->n_attention < 0 || p->n_attention > NFI_MAX_ATTENTION)
    return fail("attention_values must be in [0, 15]");
  if (!(p->scene_range > 0.f)) return fail("scene_range must be positive");
  if (!p->planes || !p->w1 || !p->b1 || !p->w2 || !p->b2 || !p->c2w)
    return fail("planes / decoder weights / tform_cam2world must be given");
  if (p->n_attention > 0 && !p->palette) return fail("palette missing (attention_values > 0)");
  if (p->use_sdf && (!p->beta || !p->alpha)) return fail("use_sdf needs beta and alpha");
  if (p->row_offset < 0 || p->full_height < 0 ||
      (p->full_height > 0 && p->row_offset + p->height > p->full_height))
    return fail("row tile outside the image (row_offset + height > full_height)");
  if (p->view_features && (!p->w3 || !p->b3))
    return fail("view_features given without w3 / b3 (ViewDirectionMapper.output)");
  if (p->noise_mode == NFI_NOISE_EXPLICIT) {
    if (!p->noise_t) return fail("noise_t missing (randomize=True)");
    if (p->fine_sampling && !p->noise_u) return fail("noise_u missing (fine_sampling)");
  } else if (p->noise_mode == NFI_NOISE_PHILOX) {
    return fail("NFI_NOISE_PHILOX is a host-entry mode: fill noise_t / noise_u with "
                "nfi_fill_uniform and pass NFI_NOISE_EXPLICIT");
  } else if (p->noise_mode != NFI_NOISE_DETERMINISTIC) {
    return fail("unknown noise_mode");
  }
  if (p->extra_mode == NFI_EXTRA_SEMANTICS && p->n_attention <= 0)
    return fail("compute_semantics needs attention_values > 0");  // run.py:232
  if (p->extra_mode < 0 || p->extra_mode > 2) return fail("unknown extra_mode");
  if (p->extra_mode != NFI_EXTRA_NONE && !p->extra) return fail("extra output buffer missing");
  if (p->compute_normals && !(p->mlp_mode & 0x1000)) {  // (0x1000: p->normals is a debug buffer)
    if (!p->use_sdf) return fail("compute_normals needs use_sdf");  // run.py:229
    if (!p->normals) return fail("normals output buffer missing");
  }
  if (!p->rgb || !p->depth || !p->mask) return fail("output buffers missing");
  return 0;
}

size_t num_ctas(const nfi_render_params* p) {
  const size_t tx = (p->width + nfi::kTileW - 1) / nfi::kTileW;
  const size_t ty = (p->height + nfi::kTileH - 1) / nfi::kTileH;
  return tx * ty * (size_t)p->batch;
}

constexpr size_t kWeightImageBytes = 32768;  // workspace header (nfi::kWiBytes rounded up)
constexpr size_t kBackwardWorkspaceBytes = 65536;  // forward + backward weight images

constexpr size_t kMaxPersistentCtas = 160;  // >= SM count of any sm_90 part (H100 SXM: 132)

// persistent pipelined kernels (nfi_pipe.cu): one CTA per SM, one scratch slab per CTA
size_t num_tc_ctas(const nfi_render_params* p) {  // persistent grid: at most one CTA per SM
  const size_t want = num_ctas(p);
  return want < kMaxPersistentCtas ? want : kMaxPersistentCtas;
}

// Can the tensor-core kernel take this configuration?
bool tc_supported(const nfi_render_params* p) {
  if (p->view_features) return false;  // view-direction conditioning (CARLA): SIMT kernels
  const int mode = p->mlp_mode & 0xff;
  const bool pipe_mode = (mode == NFI_MLP_TC_PIPE || mode == NFI_MLP_AUTO || mode == NFI_MLP_TC_WARPSPEC);
  // surface normals: a second pipelined kernel after the render (nfi_normals_pipe.cuh), which
  // walks the merged samples and so needs the forward pass's fine depths; else the SIMT kernel
  if (p->compute_normals && !(p->mlp_mode & 0x1000) &&
      !(pipe_mode && (!p->fine_sampling || p->z_fine != nullptr) && p->n_peers == 0))
    return false;
  // semantics: the pipelined kernel parks the coarse samples' probabilities; NOUT_PAD = 4 only
  // exists for palettes of <= 3 entries, kept on the SIMT kernel
  if (p->extra_mode == NFI_EXTRA_SEMANTICS && !(pipe_mode && p->n_attention > 3)) return false;
  const int smax = 64;  // lockstep kernel: per-ray columns in tile memory
  if (pipe_mode)  // pipelined kernel: <= 4 samples per lane
    return p->num_samples <= 128 && p->num_samples % 4 == 0;  // in the resampler, float4 jitter
  if (p->fine_sampling && p->num_samples > smax) return false;
  return true;
}

bool wants_normals(const nfi_render_params* p) {
  return p->compute_normals && !(p->mlp_mode & 0x1000);
}

int ne_store_of(const nfi_render_params* p) {
  return (p->extra_mode == NFI_EXTRA_SEMANTICS ? nout_pad_of(p) - 1 : 0) +
         (wants_normals(p) ? 3 : 0);
}

template <typename K>
int launch(K kernel, const nfi_render_params& p, size_t smem_bytes, cudaStream_t st) {
  if (smem_bytes > 227 * 1024)
    return fail("depth_samples_per_ray too large for the shared-memory columns");
  NFI_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)smem_bytes));
  kernel<<<(unsigned)num_ctas(&p), nfi::kThreads, smem_bytes, st>>>(p);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

template <int NP, int EX>
int launch_fwd_fine(const nfi_render_params& p, size_t smem, cudaStream_t st) {
  if (wants_normals(&p)) {
    if (p.fine_sampling) return launch(nfi::render_forward_simt<NP, EX, true, true>, p, smem, st);
    return launch(nfi::render_forward_simt<NP, EX, false, true>, p, smem, st);
  }
  if (p.fine_sampling) return launch(nfi::render_forward_simt<NP, EX, true>, p, smem, st);
  return launch(nfi::render_forward_simt<NP, EX, false>, p, smem, st);
}

template <int NP>
int launch_fwd_extra(const nfi_render_params& p, size_t smem, cudaStream_t st) {
  switch (p.extra_mode) {
    case NFI_EXTRA_COORDS: return launch_fwd_fine<NP, 1>(p, smem, st);
    case NFI_EXTRA_SEMANTICS: return launch_fwd_fine<NP, 2>(p, smem, st);
    default: return launch_fwd_fine<NP, 0>(p, smem, st);
  }
}

template <int NP, int EX>
int launch_fwd_tc_fine(const nfi_render_params& p, const unsigned char* wimg, float* scratch,
                       cudaStream_t st) {
  const int mode = p.mlp_mode & 0xff;
  if (mode == NFI_MLP_TC_PIPE || mode == NFI_MLP_AUTO || mode == NFI_MLP_TC_WARPSPEC) {
    // persistent pipelined kernel (nfi_pipe.cu): one CTA per SM, tiles strided over the grid
    int dev = 0, sms = 0;
    NFI_CUDA(cudaGetDevice(&dev));
    NFI_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    size_t grid = num_ctas(&p);
    if (grid > (size_t)sms) grid = sms;
    if (grid > kMaxPersistentCtas) grid = kMaxPersistentCtas;
    return nfi::launch_pipe_forward(p, NP, wimg, scratch, (unsigned)grid, st, g_err,
                                    sizeof(g_err));
  }
  if (p.n_peers > 0) return fail("peer outputs (n_peers > 0) need the pipelined kernel");
  if constexpr (EX == 2) {
    return fail("semantics output on tensor cores: pipelined kernel only");
  } else {
  {  // render_forward_tc: 4 tile groups per 512-thread CTA, one CTA per 2x2 tiles
    const size_t tx = (p.width + nfi::kTileW - 1) / nfi::kTileW;
    const size_t ty = (p.height + nfi::kTileH - 1) / nfi::kTileH;
    const unsigned grid = (unsigned)(((tx + 1) / 2) * ((ty + 1) / 2) * (size_t)p.batch);
    if (p.fine_sampling) {
      auto k = nfi::render_forward_tc<NP, EX, true>;
      NFI_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    nfi::kSmTcBytes));
      k<<<grid, nfi::kTcThreads, nfi::kSmTcBytes, st>>>(p, wimg, scratch);
    } else {
      auto k = nfi::render_forward_tc<NP, EX, false>;
      NFI_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    nfi::kSmTcBytes));
      k<<<grid, nfi::kTcThreads, nfi::kSmTcBytes, st>>>(p, wimg, scratch);
    }
    NFI_CUDA(cudaGetLastError());
    return 0;
  }
  }
}

int launch_fwd_tc(const nfi_render_params& p, int np, cudaStream_t st) {
  unsigned char* wimg = (unsigned char*)p.workspace;
  float* scratch = (float*)(wimg + kWeightImageBytes);
  const int nout = 1 + (p.n_attention > 0 ? p.n_attention : 3);
  const int wmode = p.mlp_mode & 0xff;
  const bool pipe = (wmode == NFI_MLP_TC_PIPE || wmode == NFI_MLP_AUTO || wmode == NFI_MLP_TC_WARPSPEC);
  if (pipe) {
    if (nfi::launch_pipe_weight_image(p, wimg, st)) return fail("weight image launch failed");
  } else {
    nfi::prep_weight_image<<<1, 256, 0, st>>>(p.w1, p.b1, p.w2, p.b2, nout, wimg, 1.f, 0.f, 1.f);
  }
  NFI_CUDA(cudaGetLastError());
  const bool coords = p.extra_mode == NFI_EXTRA_COORDS;
  const bool sem = p.extra_mode == NFI_EXTRA_SEMANTICS;  // pipelined kernel only (tc_supported)
  switch (np) {
    case 4:
      return coords ? launch_fwd_tc_fine<4, 1>(p, wimg, scratch, st)
                    : launch_fwd_tc_fine<4, 0>(p, wimg, scratch, st);
    case 12:
      if (sem) return launch_fwd_tc_fine<12, 2>(p, wimg, scratch, st);
      return coords ? launch_fwd_tc_fine<12, 1>(p, wimg, scratch, st)
                    : launch_fwd_tc_fine<12, 0>(p, wimg, scratch, st);
    default:
      if (sem) return launch_fwd_tc_fine<16, 2>(p, wimg, scratch, st);
      return coords ? launch_fwd_tc_fine<16, 1>(p, wimg, scratch, st)
                    : launch_fwd_tc_fine<16, 0>(p, wimg, scratch, st);
  }
}

// SIMT reference decoder (one point per thread), for nfi_decoder_forward
template <int NOUT_PAD>
__global__ void __launch_bounds__(128)
decoder_forward_simt(const float* __restrict__ feats, long long n, int nout,
                     const float* __restrict__ w1, const float* __restrict__ b1,
                     const float* __restrict__ w2, const float* __restrict__ b2,
                     float* __restrict__ outp) {
  __shared__ __align__(16) float W1t[nfi::kC * nfi::kHid];
  __shared__ __align__(16) float b1s[nfi::kHid];
  __shared__ __align__(16) float W2t[nfi::kHid * NOUT_PAD];
  __shared__ __align__(16) float b2s[NOUT_PAD];
  for (int i = threadIdx.x; i < nfi::kC * nfi::kHid; i += 128)
    W1t[i] = w1[(i % nfi::kHid) * nfi::kC + i / nfi::kHid];
  for (int i = threadIdx.x; i < nfi::kHid; i += 128) b1s[i] = b1[i];
  for (int i = threadIdx.x; i < nfi::kHid * NOUT_PAD; i += 128) {
    const int j = i / NOUT_PAD, o = i % NOUT_PAD;
    W2t[i] = (o < nout) ? w2[o * nfi::kHid + j] : 0.f;
  }
  for (int i = threadIdx.x; i < NOUT_PAD; i += 128) b2s[i] = (i < nout) ? b2[i] : 0.f;
  __syncthreads();
  const long long row = (long long)blockIdx.x * 128 + threadIdx.x;
  if (row >= n) return;
  float out[NOUT_PAD];
  float h[nfi::kHid];
  nfi::mlp_forward<NOUT_PAD, false>(feats + row * nfi::kC, W1t, b1s, W2t, b2s, out, h);
  for (int o = 0; o < NOUT_PAD; ++o)
    if (o < nout) outp[row * nout + o] = out[o];
}

// ---------------------------------------------------------------- device-side noise
// Philox-4x32-10 (Salmon et al., SC'11), one counter -> four uniforms.
__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
  const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
  const uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
  c[0] = hi1 ^ c[1] ^ k0;
  c[1] = lo1;
  c[2] = hi0 ^ c[3] ^ k1;
  c[3] = lo0;
}
__global__ void __launch_bounds__(256)
fill_uniform_kernel(float* __restrict__ dst, long long n, unsigned long long seed,
                    unsigned stream_id, long long offset) {
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // group of 4 outputs
  if (4 * i4 >= n) return;
  const unsigned long long ctr = (unsigned long long)(offset / 4 + i4);
  uint32_t c[4] = {(uint32_t)ctr, (uint32_t)(ctr >> 32), stream_id, 0u};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = (float)(c[j] >> 8) * (1.0f / 16777216.0f);
  if (4 * i4 + 3 < n) {
    *reinterpret_cast<float4*>(dst + 4 * i4) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    for (int j = 0; j < 4 && 4 * i4 + j < n; ++j) dst[4 * i4 + j] = v[j];
  }
}

// ---------------------------------------------------------------- re-layout
// [B,32,R,R] x3 (channel-first)  ->  [B,3,R,R,32] (channel-last), and back.
// 32 channels x 32 pixels per block through a padded shared tile: both the
// reads (along pixels) and the writes (along channels) are 128-byte lines.
__global__ void __launch_bounds__(256)
planes_to_cl_kernel(const float* __restrict__ xy, const float* __restrict__ xz,
                    const float* __restrict__ yz, long long batch_stride, int RR,
                    float* __restrict__ dst) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, pl = blockIdx.y;
  const float* src = (pl == 0 ? xy : (pl == 1 ? xz : yz)) + (long long)b * batch_stride;
  const int pix0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int c = ty; c < 32; c += 8) {
    const int pix = pix0 + tx;
    tile[c][tx] = (pix < RR) ? src[(long long)c * RR + pix] : 0.f;
  }
  __syncthreads();
  float* out = dst + ((long long)(b * 3 + pl) * RR) * 32;
  for (int q = ty; q < 32; q += 8) {
    const int pix = pix0 + q;
    if (pix < RR) out[(long long)pix * 32 + tx] = tile[tx][q];
  }
}

__global__ void __launch_bounds__(256)
planes_from_cl_kernel(const float* __restrict__ src, int RR, float* __restrict__ dst) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, pl = blockIdx.y;
  const float* in = src + ((long long)(b * 3 + pl) * RR) * 32;
  float* out = dst + ((long long)(b * 3 + pl) * 32) * RR;
  const int pix0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int q = ty; q < 32; q += 8) {
    const int pix = pix0 + q;
    tile[q][tx] = (pix < RR) ? in[(long long)pix * 32 + tx] : 0.f;
  }
  __syncthreads();
  for (int c = ty; c < 32; c += 8) {
    const int pix = pix0 + tx;
    if (pix < RR) out[(long long)c * RR + pix] = tile[tx][c];
  }
}

}  // namespace

extern "C" {

int nfi_abi_version(void) { return NFI_ABI_VERSION; }

const char* nfi_build_info(void) {
  return "libnfi_render sm_90a (compute_90a) nvcc " NFI_STR(__CUDACC_VER_MAJOR__) "." NFI_STR(
      __CUDACC_VER_MINOR__) " fmad=false";
}

const char* nfi_last_error(void) { return g_err; }

size_t nfi_render_workspace_bytes(const nfi_render_params* p) {
  if (p == nullptr) return 0;
  size_t fwd = 0;
  if (p->fine_sampling) {
    // scratch for the coarse samples, sized for the kernel that will run
    const int mode = p->mlp_mode & 0xff;
    const bool pipe_mode =
        (mode == NFI_MLP_TC_PIPE || mode == NFI_MLP_AUTO || mode == NFI_MLP_TC_WARPSPEC);
    if (pipe_mode && tc_supported(p)) {  // persistent: one slab per CTA (<= one per SM)
      fwd = num_tc_ctas(p) * nfi::pipe_scratch_bytes_per_cta(
                                 p->num_samples,
                                 p->extra_mode == NFI_EXTRA_SEMANTICS ? nout_pad_of(p) - 1 : 0);
    } else if (mode == NFI_MLP_TC_3XTF32) {  // lockstep: one slab per tile group of every CTA
      const size_t tx = (p->width + nfi::kTileW - 1) / nfi::kTileW;
      const size_t ty = (p->height + nfi::kTileH - 1) / nfi::kTileH;
      fwd = ((tx + 1) / 2) * ((ty + 1) / 2) * (size_t)p->batch * nfi::kGroups *
            nfi::pipe_scratch_bytes_per_cta(p->num_samples, 0);
    } else {  // fp32 SIMT kernel: one slab per CTA (= tile)
      fwd = num_ctas(p) * nfi::fwd_scratch_floats_per_cta(p->num_samples, ne_store_of(p)) *
            sizeof(float);
    }
  }
  // (+ the backward weight image of the normals kernel, behind the scratch)
  return kWeightImageBytes + fwd + 256 + (wants_normals(p) && tc_supported(p) ? 32768 : 0);
}

int nfi_planes_to_channel_last(const float* xy, const float* xz, const float* yz,
                               int64_t batch_stride, int32_t batch, int32_t plane_res, float* dst,
                               void* stream) {
  if (!xy || !xz || !yz || !dst || batch <= 0 || plane_res <= 0) return fail("bad re-layout args");
  const int RR = plane_res * plane_res;
  dim3 grid((RR + 31) / 32, 3, batch);
  planes_to_cl_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(xy, xz, yz, batch_stride, RR, dst);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int nfi_planes_from_channel_last(const float* src, int32_t batch, int32_t plane_res, float* dst,
                                 void* stream) {
  if (!src || !dst || batch <= 0 || plane_res <= 0) return fail("bad re-layout args");
  const int RR = plane_res * plane_res;
  dim3 grid((RR + 31) / 32, 3, batch);
  planes_from_cl_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, RR, dst);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int nfi_fill_uniform(float* dst, int64_t n, uint64_t seed, uint32_t stream_id, int64_t offset,
                     void* stream) {
  if (!dst || n < 0 || offset < 0 || (offset & 3) || ((uintptr_t)dst & 15))
    return fail("nfi_fill_uniform: dst must be 16-byte aligned, offset a multiple of 4");
  if (n == 0) return 0;
  const long long groups = (n + 3) / 4;
  fill_uniform_kernel<<<(unsigned)((groups + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      dst, n, seed, stream_id, offset);
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int nfi_render_forward(const nfi_render_params* params, void* stream) {
  if (int rc = check_params(params)) return rc;
  const nfi_render_params& p = *params;
  const int np = nout_pad_of(params);
  cudaStream_t st = (cudaStream_t)stream;
  const int mode = p.mlp_mode & 0xff;
  if ((mode == NFI_MLP_TC_3XTF32 || mode == NFI_MLP_TC_WARPSPEC || mode == NFI_MLP_TC_PIPE) &&
      !tc_supported(params))
    return fail("tensor-core modes need S <= 128 and S % 4 == 0 (lockstep kernel: S <= 64) and "
                "no semantics output; use NFI_MLP_AUTO");
  const bool want_tc = mode == NFI_MLP_TC_3XTF32 || mode == NFI_MLP_TC_WARPSPEC ||
                       mode == NFI_MLP_TC_PIPE ||
                       (mode == NFI_MLP_AUTO && tc_supported(params));
  if (want_tc || p.fine_sampling) {
    if (!p.workspace || p.workspace_bytes < nfi_render_workspace_bytes(params))
      return fail("workspace too small (see nfi_render_workspace_bytes)");
  }
  if (p.n_peers < 0 || p.n_peers > NFI_MAX_PEERS) return fail("n_peers out of range");
  for (int q = 0; q < p.n_peers; ++q)
    if (!p.peer_rgb[q] || !p.peer_depth[q] || !p.peer_mask[q]) return fail("peer output pointer is NULL");
  if (want_tc) {
    if (int rc = launch_fwd_tc(p, np, st)) return rc;
    if (wants_normals(params)) {
      int dev = 0, sms = 0;
      NFI_CUDA(cudaGetDevice(&dev));
      NFI_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
      size_t grid = num_ctas(&p);
      if (grid > (size_t)sms) grid = sms;
      unsigned char* ws = (unsigned char*)p.workspace;
      const size_t off = (nfi_render_workspace_bytes(params) - 32768) & ~(size_t)255;
      return nfi::launch_pipe_normals(p, np, ws, ws + off, (unsigned)grid, st, g_err, sizeof(g_err));
    }
    return 0;
  }
  if (p.n_peers > 0) return fail("peer outputs (n_peers > 0) need the pipelined kernel");
  if (p.view_features) {
    nfi_render_params pv = p;  // SIMT scratch starts after the weight-image header
    if (pv.workspace) pv.workspace = (unsigned char*)pv.workspace + kWeightImageBytes;
    return nfi::launch_forward_viewdir(pv, np, wants_normals(params), st, g_err, sizeof(g_err));
  }
  const size_t smem =
      nfi::fwd_smem_floats(np, p.num_samples, p.fine_sampling != 0, wants_normals(params)) *
      sizeof(float);
  nfi_render_params ps = p;  // SIMT scratch starts after the weight-image header
  if (ps.workspace) ps.workspace = (unsigned char*)ps.workspace + kWeightImageBytes;
  switch (np) {
    case 4: return launch_fwd_extra<4>(ps, smem, st);
    case 12: return launch_fwd_extra<12>(ps, smem, st);
    default: return launch_fwd_extra<16>(ps, smem, st);
  }
}

int nfi_decoder_forward(const float* features, int64_t n_points, const float* w1, const float* b1,
                        const float* w2, const float* b2, int32_t n_attention, float* out,
                        int32_t mlp_mode, void* workspace, void* stream) {
  if (!features || !w1 || !b1 || !w2 || !b2 || !out || n_points <= 0)
    return fail("bad decoder arguments");
  if (n_attention < 0 || n_attention > NFI_MAX_ATTENTION) return fail("attention_values out of range");
  const int nout = 1 + (n_attention > 0 ? n_attention : 3);
  const int np = nout <= 4 ? 4 : (nout <= 12 ? 12 : 16);
  cudaStream_t st = (cudaStream_t)stream;
  if (mlp_mode == NFI_MLP_FP32_SIMT) {
    const unsigned grid = (unsigned)((n_points + 127) / 128);
    if (np == 4) decoder_forward_simt<4><<<grid, 128, 0, st>>>(features, n_points, nout, w1, b1, w2, b2, out);
    else if (np == 12) decoder_forward_simt<12><<<grid, 128, 0, st>>>(features, n_points, nout, w1, b1, w2, b2, out);
    else decoder_forward_simt<16><<<grid, 128, 0, st>>>(features, n_points, nout, w1, b1, w2, b2, out);
    NFI_CUDA(cudaGetLastError());
    return 0;
  }
  if (!workspace) return fail("decoder (tensor-core mode) needs a 32 KiB workspace");
  unsigned char* wimg = (unsigned char*)workspace;
  nfi::prep_weight_image<<<1, 256, 0, st>>>(w1, b1, w2, b2, nout, wimg, 1.f, 0.f, 1.f);
  NFI_CUDA(cudaGetLastError());
  const long long tiles = (n_points + 127) / 128;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const unsigned grid = (unsigned)((tiles + nfi::kGroups - 1) / nfi::kGroups < sms
                                       ? (tiles + nfi::kGroups - 1) / nfi::kGroups
                                       : sms);
#define NFI_DEC(NP)                                                                          \
  do {                                                                                       \
    NFI_CUDA(cudaFuncSetAttribute(nfi::decoder_forward_tc<NP>,                               \
                                  cudaFuncAttributeMaxDynamicSharedMemorySize,               \
                                  nfi::kSmTcBytes));                                         \
    nfi::decoder_forward_tc<NP><<<grid, nfi::kTcThreads, nfi::kSmTcBytes, st>>>(             \
        features, n_points, nout, wimg, out);                                                \
  } while (0)
  if (np == 4) NFI_DEC(4); else if (np == 12) NFI_DEC(12); else NFI_DEC(16);
#undef NFI_DEC
  NFI_CUDA(cudaGetLastError());
  return 0;
}

int nfi_render_backward(const nfi_render_params* params, const nfi_render_grads* grads,
                        void* stream) {
  if (int rc = check_params(params)) return rc;
  if (grads == nullptr || grads->g_rgb == nullptr) return fail("grads->g_rgb missing");
  const nfi_render_params& p = *params;
  const nfi_render_grads& g = *grads;
  cudaStream_t st = (cudaStream_t)stream;
  // Tensor-core backward (nfi_backward_pipe.cuh): frozen decoder weights (the inversion
  // setting, run.py:628-629), no semantics output, S within the pipelined kernels' envelope,
  // and a workspace for the two weight images.  Everything else: render_backward_simt.
  const int mode = p.mlp_mode & 0xff;
  if (p.view_features)
    return nfi::launch_backward_viewdir(p, g, nout_pad_of(params), st, g_err, sizeof(g_err));
  if (g.grad_view_features || g.grad_w3 || g.grad_b3)
    return fail("grad_view_features / grad_w3 / grad_b3 need params->view_features");
  const bool wgrad = g.grad_w1 || g.grad_b1 || g.grad_w2 || g.grad_b2;
  const bool tc_env = mode != NFI_MLP_FP32_SIMT && p.extra_mode != NFI_EXTRA_SEMANTICS &&
                      p.num_samples <= 128 && p.num_samples % 4 == 0 && p.workspace != nullptr &&
                      p.workspace_bytes >= kBackwardWorkspaceBytes &&
                      (!p.fine_sampling || p.z_fine != nullptr) && g.out_rgb && g.out_mask &&
                      (!g.g_extra || g.out_extra) &&
                      ((g.grad_origins == nullptr) == (g.grad_dirs == nullptr));
  // decoder-weight gradients (the GAN generator step, run.py:1044) on the tensor cores too: a second
  // kernel (render_wgrad_pipe) beside render_backward_pipe, which then sees a frozen decoder.
  // An upstream gradient of the coords output stays on the SIMT kernel.
  const bool tc_ok = tc_env && (!wgrad || (!g.g_extra &&
                                           p.workspace_bytes >= nfi::pipe_wgrad_workspace_bytes(
                                                                    (unsigned)kMaxPersistentCtas)));
  if (tc_ok) {
    int dev = 0, sms = 0;
    NFI_CUDA(cudaGetDevice(&dev));
    NFI_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    size_t grid = num_ctas(&p);
    if (grid > (size_t)sms) grid = sms;
    if (grid > kMaxPersistentCtas) grid = kMaxPersistentCtas;  // (the wgrad workspace is sized for it)
    nfi_render_grads g1 = g;
    g1.grad_w1 = g1.grad_b1 = g1.grad_w2 = g1.grad_b2 = nullptr;
    const bool others = g1.grad_planes || g1.grad_palette || g1.grad_beta || g1.grad_alpha ||
                        g1.grad_origins;
    // The generator step (decoder gradients, cameras are data): ONE sweep, render_wgrad_pipe with
    // the plane scatter folded in.  With a pose gradient too: render_backward_pipe beside it.
    // (mlp_mode bit 0x2000: timing experiments, tools/time_wgrad.py -- two sweeps anyway)
    const bool one_sweep = wgrad && others && !g.grad_origins && !(p.mlp_mode & 0x2000);
    if ((others && !one_sweep) || !wgrad) {
      if (int rc = nfi::launch_pipe_backward(p, g1, nout_pad_of(params), (unsigned char*)p.workspace,
                                             (unsigned)grid, st, g_err, sizeof(g_err)))
        return rc;
    }
    if (wgrad)
      return nfi::launch_pipe_wgrad(p, g, nout_pad_of(params), (unsigned char*)p.workspace,
                                    (unsigned)grid, one_sweep, st, g_err, sizeof(g_err));
    return 0;
  }
  return nfi::launch_backward(*params, *grads, st, g_err, sizeof(g_err));
}

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
  return nfi::launch_sample_field(p, *sp, nout_pad_of(&p), (cudaStream_t)stream, g_err,
                                  sizeof(g_err));
}

int nfi_pose_to_matrix(const float* z0, const float* t2, const float* s, const float* q,
                       int32_t camera_flipped, int32_t batch, float* c2w, float* focal,
                       void* stream) {
  if (batch <= 0) return fail("empty batch");
  if (!t2 || !s || !q || !c2w) return fail("t2 / s / q / c2w must be given");
  if (z0 && !focal) return fail("perspective pose (z0 given) needs the focal output");
  return nfi::launch_pose_to_matrix(z0, t2, s, q, camera_flipped, batch, c2w, focal,
                                    (cudaStream_t)stream, g_err, sizeof(g_err));
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
                                             g_z0, g_t2, g_s, g_q, (cudaStream_t)stream, g_err,
                                             sizeof(g_err));
}

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
  return nfi::heads::launch_forward(*params, (cudaStream_t)stream, g_err, sizeof(g_err));
}

int nfi_sdf_points_backward(const nfi_sdf_points_params* params, const nfi_sdf_points_grads* grads,
                            void* stream) {
  if (const int rc = check_sdf_points(params)) return rc;
  if (grads == nullptr) return fail("grads is NULL");
  if (!grads->g_d && !grads->g_grad) return fail("no upstream gradient");
  if (grads->grad_w1 && (!grads->grad_b1 || !grads->grad_w2_row0 || !grads->grad_b2_0))
    return fail("decoder gradients come as a set: grad_w1, grad_b1, grad_w2_row0, grad_b2_0");
  return nfi::heads::launch_backward(*params, *grads, (cudaStream_t)stream, g_err, sizeof(g_err));
}

size_t nfi_synthesis_workspace_bytes(const nfi_synth_params* params) {
  if (params == nullptr) return 0;
  return nfi::synth::workspace_bytes(*params);
}

int nfi_synthesis_forward(const nfi_synth_params* params, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  if (params->batch <= 0) return fail("empty batch");
  return nfi::synth::forward(*params, (cudaStream_t)stream, g_err, sizeof(g_err));
}

size_t nfi_synthesis_saved_workspace_bytes(const nfi_synth_params* params) {
  if (params == nullptr) return 0;
  return nfi::synth::saved_workspace_bytes(*params);
}

int nfi_synthesis_forward_saved(const nfi_synth_params* params, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  if (params->batch <= 0) return fail("empty batch");
  return nfi::synth::forward_saved(*params, (cudaStream_t)stream, g_err, sizeof(g_err));
}

int nfi_synthesis_backward(const nfi_synth_params* params, const nfi_synth_grads* grads, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  if (grads == nullptr) return fail("grads is NULL");
  if (params->batch <= 0) return fail("empty batch");
  return nfi::synth::backward(*params, *grads, (cudaStream_t)stream, g_err, sizeof(g_err));
}

size_t nfi_synthesis_param_workspace_bytes(const nfi_synth_params* params) {
  if (params == nullptr) return 0;
  return nfi::synth::param_workspace_bytes(*params);
}

int nfi_synthesis_backward_params(const nfi_synth_params* params, const nfi_synth_grads* grads,
                                  const nfi_synth_param_grads* param_grads, void* stream) {
  if (params == nullptr) return fail("params is NULL");
  if (grads == nullptr) return fail("grads is NULL");
  if (param_grads == nullptr) return fail("param_grads is NULL");
  if (params->batch <= 0) return fail("empty batch");
  return nfi::synth::backward_params(*params, *grads, *param_grads, (cudaStream_t)stream, g_err,
                                     sizeof(g_err));
}

int nfi_render_forward_host(const nfi_render_params* hp, int32_t device) {
  // Host buffers in, host buffers out.  The batch is cut into chunks of images
  // (images are independent: SURVEY.md section 8e) and pipelined over two
  // streams: while chunk c is re-laid-out and rendered, chunk c+1's planes and
  // noise are already crossing PCIe, and chunk c-1's rgb/depth/mask go back.
  if (hp == nullptr) return fail("params is NULL");
  if (hp->view_features)
    return fail("view-direction conditioning is not offered through the host entry point "
                "(use nfi_render_forward)");
  NFI_CUDA(cudaSetDevice(device));
  cudaStream_t st = nullptr, cp = nullptr;
  // Everything acquired below is released on the single exit path at the bottom (streams,
  // events, stream-ordered allocations) and the one process-wide setting this function
  // touches -- the release threshold of the device's default memory pool, raised so that the
  // per-call buffers are recycled instead of returned to the driver -- is put back.
  cudaMemPool_t pool = nullptr;
  uint64_t old_keep = 0;
  bool pool_changed = false;
  {
    cudaError_t e0 = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    if (e0 == cudaSuccess) e0 = cudaStreamCreateWithFlags(&cp, cudaStreamNonBlocking);
    if (e0 == cudaSuccess) e0 = cudaDeviceGetDefaultMemPool(&pool, device);
    if (e0 == cudaSuccess)
      e0 = cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &old_keep);
    if (e0 == cudaSuccess) {
      uint64_t keep = UINT64_MAX;
      e0 = cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
      pool_changed = (e0 == cudaSuccess);
    }
    if (e0 != cudaSuccess) {
      if (pool_changed) cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &old_keep);
      if (cp) cudaStreamDestroy(cp);
      if (st) cudaStreamDestroy(st);
      snprintf(g_err, sizeof(g_err), "host entry point set-up failed: %s", cudaGetErrorString(e0));
      return 2;
    }
  }

  nfi_render_params d = *hp;
  const size_t B = hp->batch, H = hp->height, W = hp->width, S = hp->num_samples;
  const size_t R = hp->plane_res, A = hp->n_attention;
  const size_t nout = 1 + (A > 0 ? A : 3);
  const size_t rays_img = H * W, n_rays = B * rays_img;
  void* to_free[40];
  int n_free = 0;
  int rc = 0;
  auto dalloc = [&](size_t bytes) -> float* {
    void* q = nullptr;
    if (cudaMallocAsync(&q, bytes ? bytes : 4, st) != cudaSuccess) return nullptr;
    to_free[n_free++] = q;
    return (float*)q;
  };
  auto up = [&](const float* h, size_t n) -> const float* {  // small tensors: compute stream
    if (h == nullptr) return nullptr;
    float* q = dalloc(n * sizeof(float));
    if (q) cudaMemcpyAsync(q, h, n * sizeof(float), cudaMemcpyHostToDevice, st);
    return q;
  };
  // chunk = 8 images: 128 CTAs of the lockstep kernel, ~34 MB per image on the wire
  const size_t CB = B < 8 ? B : 8;
  const size_t n_chunks = (B + CB - 1) / CB;
  const size_t plane_img = 3 * R * R * 32;
  float* planes_cf = dalloc(B * plane_img * sizeof(float));
  float* planes_cl = dalloc(B * plane_img * sizeof(float));
  const bool philox = hp->noise_mode == NFI_NOISE_PHILOX;
  const bool has_nt = philox || (hp->noise_mode == NFI_NOISE_EXPLICIT && hp->noise_t);
  const bool has_nu = has_nt && hp->fine_sampling && (philox || hp->noise_u);
  if (philox) d.noise_mode = NFI_NOISE_EXPLICIT;
  float* noise_t = has_nt ? dalloc(n_rays * S * sizeof(float)) : nullptr;
  float* noise_u = has_nu ? dalloc(n_rays * S * sizeof(float)) : nullptr;
  d.w1 = up(hp->w1, 64 * 32);
  d.b1 = up(hp->b1, 64);
  d.w2 = up(hp->w2, nout * 64);
  d.b2 = up(hp->b2, nout);
  const float* palette = up(hp->palette, B * A * 3);
  d.beta = up(hp->beta, 1);
  d.alpha = up(hp->alpha, 1);
  const float* c2w = up(hp->c2w, B * 16);
  const float* focal = up(hp->focal, B);
  const float* center = up(hp->center, B * 2);
  const float* bbox = up(hp->bbox, B * 4);
  const size_t ne = hp->extra_mode == NFI_EXTRA_COORDS ? 3 : (hp->extra_mode ? A : 0);
  float* rgb = dalloc(n_rays * 3 * sizeof(float));
  float* depth = dalloc(n_rays * sizeof(float));
  float* mask = dalloc(n_rays * sizeof(float));
  float* extra = ne ? dalloc(n_rays * ne * sizeof(float)) : nullptr;
  d.normals = (hp->compute_normals && hp->normals) ? dalloc(n_rays * 3 * sizeof(float)) : nullptr;
  float* normals = d.normals;
  d.z_fine = nullptr;
  d.batch = (int32_t)CB;
  d.workspace_bytes = nfi_render_workspace_bytes(&d);
  d.workspace = dalloc(d.workspace_bytes);
  cudaEvent_t ready[64];
  size_t n_events = 0;
  if (!planes_cf || !planes_cl || !rgb || !depth || !mask || !d.workspace || n_chunks > 64 ||
      (has_nt && !noise_t) || (has_nu && !noise_u)) {
    rc = fail(n_chunks > 64 ? "batch too large for the host entry point (max 512 images)"
                            : "device allocation failed");
  } else {
    // the copy stream may only touch the buffers once their allocation (on st) is done
    cudaEvent_t alloc_done = nullptr;
    if (cudaEventCreateWithFlags(&alloc_done, cudaEventDisableTiming) != cudaSuccess) {
      rc = fail("cudaEventCreate failed");
    } else {
      cudaEventRecord(alloc_done, st);
      cudaStreamWaitEvent(cp, alloc_done, 0);
      cudaEventDestroy(alloc_done);
    }
    for (size_t c = 0; c < n_chunks && !rc; ++c) {
      const size_t b0 = c * CB, nb = (b0 + CB <= B) ? CB : B - b0;
      cudaMemcpyAsync(planes_cf + b0 * plane_img, hp->planes + b0 * plane_img,
                      nb * plane_img * sizeof(float), cudaMemcpyHostToDevice, cp);
      if (has_nt && !philox)
        cudaMemcpyAsync(noise_t + b0 * rays_img * S, hp->noise_t + b0 * rays_img * S,
                        nb * rays_img * S * sizeof(float), cudaMemcpyHostToDevice, cp);
      if (has_nu && !philox)
        cudaMemcpyAsync(noise_u + b0 * rays_img * S, hp->noise_u + b0 * rays_img * S,
                        nb * rays_img * S * sizeof(float), cudaMemcpyHostToDevice, cp);
      cudaEventCreateWithFlags(&ready[c], cudaEventDisableTiming);
      n_events = c + 1;
      cudaEventRecord(ready[c], cp);
      cudaStreamWaitEvent(st, ready[c], 0);
      nfi_render_params q = d;
      q.batch = (int32_t)nb;
      q.planes = planes_cl + b0 * plane_img;
      q.palette = palette ? palette + b0 * A * 3 : nullptr;
      q.c2w = c2w + b0 * 16;
      q.focal = focal ? focal + b0 : nullptr;
      q.center = center ? center + b0 * 2 : nullptr;
      q.bbox = bbox ? bbox + b0 * 4 : nullptr;
      q.noise_t = has_nt ? noise_t + b0 * rays_img * S : nullptr;
      q.noise_u = has_nu ? noise_u + b0 * rays_img * S : nullptr;
      q.rgb = rgb + b0 * rays_img * 3;
      q.depth = depth + b0 * rays_img;
      q.mask = mask + b0 * rays_img;
      q.extra = extra ? extra + b0 * rays_img * ne : nullptr;
      q.normals = normals ? normals + b0 * rays_img * 3 : nullptr;
      if (philox) {  // the two draws of the path, generated where the reference draws them
        const int64_t off = (int64_t)(b0 * rays_img * S), cnt = (int64_t)(nb * rays_img * S);
        rc = nfi_fill_uniform(noise_t + off, cnt, hp->noise_seed, 0u, off, st);
        if (!rc && has_nu) rc = nfi_fill_uniform(noise_u + off, cnt, hp->noise_seed, 1u, off, st);
        if (rc) break;
      }
      const float* cf = planes_cf + b0 * plane_img;
      rc = nfi_planes_to_channel_last(cf, cf + 32 * R * R, cf + 64 * R * R, (int64_t)(96 * R * R),
                                      (int32_t)nb, (int32_t)R, planes_cl + b0 * plane_img, st);
      if (!rc) rc = nfi_render_forward(&q, st);
      if (!rc) {
        cudaMemcpyAsync(hp->rgb + b0 * rays_img * 3, q.rgb, nb * rays_img * 3 * sizeof(float),
                        cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(hp->depth + b0 * rays_img, q.depth, nb * rays_img * sizeof(float),
                        cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(hp->mask + b0 * rays_img, q.mask, nb * rays_img * sizeof(float),
                        cudaMemcpyDeviceToHost, st);
        if (ne && hp->extra)
          cudaMemcpyAsync(hp->extra + b0 * rays_img * ne, q.extra,
                          nb * rays_img * ne * sizeof(float), cudaMemcpyDeviceToHost, st);
        if (normals)
          cudaMemcpyAsync(hp->normals + b0 * rays_img * 3, q.normals,
                          nb * rays_img * 3 * sizeof(float), cudaMemcpyDeviceToHost, st);
      }
    }
  }
  cudaError_t e1 = cudaStreamSynchronize(cp);
  for (int i = 0; i < n_free; ++i) cudaFreeAsync(to_free[i], st);
  cudaError_t e = cudaStreamSynchronize(st);
  for (size_t c = 0; c < n_events; ++c) cudaEventDestroy(ready[c]);
  cudaStreamDestroy(cp);
  cudaStreamDestroy(st);
  if (pool_changed) cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &old_keep);
  if (e == cudaSuccess) e = e1;
  if (!rc && e != cudaSuccess) {
    snprintf(g_err, sizeof(g_err), "render failed: %s", cudaGetErrorString(e));
    rc = 2;
  }
  return rc;
}

}  // extern "C"
