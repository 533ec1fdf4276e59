// C-ABI entry points of libnfi_render.so (see include/nfi_render.h).
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a --fmad=false -lineinfo
//        (nerf_from_image_b200/csrc/build.sh).  No torch, no CPU fallback: on a
//        machine without an sm_90 device every launch returns an error.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>

#include "nfi_backward.cuh"
#include "nfi_weight_image.cuh"
#include "nfi_pipe_launch.h"
#include "nfi_render.h"
#include "nfi_route.h"

#define NFI_STR_(x) #x
#define NFI_STR(x) NFI_STR_(x)

using nfi::fail;

namespace {

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
  if (nfi::wants_normals(*p)) {
    if (!p->use_sdf) return fail("compute_normals needs use_sdf");  // run.py:229
    if (!p->normals) return fail("normals output buffer missing");
  }
  if (!p->rgb || !p->depth || !p->mask) return fail("output buffers missing");
  return 0;
}

// the SM count of the current device
int sm_count(int* sms) {
  int dev = 0;
  NFI_CUDA(cudaGetDevice(&dev));
  NFI_CUDA(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
  return 0;
}

// persistent pipelined kernels (nfi_pipe.cu): one CTA per SM, one scratch slab per CTA, at most
// kMaxPersistentCtas (the workspace sizes assume no more)
size_t num_tc_ctas(const nfi_render_params& p) {
  const size_t want = nfi::num_tiles(p);
  return want < nfi::kMaxPersistentCtas ? want : nfi::kMaxPersistentCtas;
}

// the grid of a persistent pipelined launch: num_tc_ctas, and no more CTAs than this device's SMs
int persistent_grid(const nfi_render_params& p, unsigned* grid) {
  int sms = 0;
  if (int rc = sm_count(&sms)) return rc;
  const size_t want = num_tc_ctas(p);
  *grid = (unsigned)(want < (size_t)sms ? want : (size_t)sms);
  return 0;
}

bool is_pipe(nfi::Route r) { return r == nfi::Route::kPipe || r == nfi::Route::kPipeVd; }

// Byte offsets in the forward's workspace (nfi_layout.h): the scratch slabs behind the weight
// image, the backward image of the normals kernel behind the scratch, and the total size.
struct FwdWorkspace {
  size_t scratch, normals_image, total;
};
FwdWorkspace fwd_workspace(const nfi_render_params& p, const nfi::Plan& r) {
  const int nes = p.extra_mode == NFI_EXTRA_SEMANTICS ? nfi::nout_pad_of(p.n_attention) - 1 : 0;
  size_t slabs = 0;
  if (p.fine_sampling) {  // the coarse samples, one slab per CTA of the kernel that will run
    if (is_pipe(r.route))
      slabs = num_tc_ctas(p) * nfi::pipe_scratch_bytes_per_cta(p.num_samples, nes);
    else  // the SIMT kernel parks the normals as three more extras
      slabs = nfi::num_tiles(p) * sizeof(float) *
              nfi::fwd_scratch_floats_per_cta(p.num_samples, nes + (nfi::wants_normals(p) ? 3 : 0));
  }
  FwdWorkspace w;
  w.scratch = p.view_features ? nfi::kVdFwdImageSlot : nfi::kFwdImageSlot;
  const size_t end = w.scratch + slabs + 256;
  w.normals_image = end & ~(size_t)255;
  w.total = end + (r.normals_pipe ? nfi::kBwdImageBytes : 0);
  return w;
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

// the text behind nfi_last_error, one per host thread
thread_local char g_err[512] = "";

}  // namespace

int nfi::fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}

extern "C" {

int nfi_abi_version(void) { return NFI_ABI_VERSION; }

const char* nfi_build_info(void) {
  return "libnfi_render sm_90a (compute_90a) nvcc " NFI_STR(__CUDACC_VER_MAJOR__) "." NFI_STR(
      __CUDACC_VER_MINOR__) " fmad=false";
}

const char* nfi_last_error(void) { return g_err; }

size_t nfi_render_workspace_bytes(const nfi_render_params* p) {
  if (p == nullptr) return 0;
  return fwd_workspace(*p, nfi::route_forward(*p)).total;
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
  cudaStream_t st = (cudaStream_t)stream;
  if (p.n_peers < 0 || p.n_peers > NFI_MAX_PEERS) return fail("n_peers out of range");
  for (int q = 0; q < p.n_peers; ++q)
    if (!p.peer_rgb[q] || !p.peer_depth[q] || !p.peer_mask[q]) return fail("peer output pointer is NULL");
  const nfi::Plan r = nfi::route_forward(p);
  if (r.route == nfi::Route::kRefused) return fail("%s", r.refusal);
  const FwdWorkspace ws = fwd_workspace(p, r);
  if ((is_pipe(r.route) || p.fine_sampling) && (!p.workspace || p.workspace_bytes < ws.total))
    return fail("workspace too small (see nfi_render_workspace_bytes)");
  unsigned char* wsp = (unsigned char*)p.workspace;
  if (!is_pipe(r.route)) {
    nfi_render_params ps = p;  // SIMT scratch starts after the weight-image header
    if (ps.workspace) ps.workspace = wsp + ws.scratch;
    if (r.route == nfi::Route::kSimtVd)
      return nfi::launch_forward_simt<true>(ps, nfi::wants_normals(p), st);
    return nfi::launch_forward_simt<false>(ps, nfi::wants_normals(p), st);
  }
  unsigned grid = 0;
  if (int rc = persistent_grid(p, &grid)) return rc;
  float* scratch = (float*)(wsp + ws.scratch);
  const int rc = r.route == nfi::Route::kPipeVd
                     ? nfi::launch_pipe_forward<true>(p, wsp, scratch, grid, st)
                     : nfi::launch_pipe_forward<false>(p, wsp, scratch, grid, st);
  if (rc || !r.normals_pipe) return rc;
  return nfi::launch_pipe_normals(p, wsp, wsp + ws.normals_image, grid, st);
}

int nfi_decoder_forward(const float* features, int64_t n_points, const float* w1, const float* b1,
                        const float* w2, const float* b2, int32_t n_attention, float* out,
                        int32_t mlp_mode, void* workspace, void* stream) {
  if (!features || !w1 || !b1 || !w2 || !b2 || !out || n_points <= 0)
    return fail("bad decoder arguments");
  if (n_attention < 0 || n_attention > NFI_MAX_ATTENTION) return fail("attention_values out of range");
  const int nout = nfi::nout_of(n_attention), np = nfi::nout_pad_of(n_attention);
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
  int sms = 0;
  if (int rc = sm_count(&sms)) return rc;
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
  if (p.fine_sampling && p.z_fine == nullptr)
    return fail("backward needs the z_fine buffer the forward pass filled");
  if (!g.out_rgb || !g.out_mask) return fail("backward needs the forward outputs (out_rgb, out_mask)");
  if (g.g_extra && !g.out_extra) return fail("g_extra given without out_extra");
  if ((g.grad_origins == nullptr) != (g.grad_dirs == nullptr))
    return fail("grad_origins and grad_dirs must be given together");
  cudaStream_t st = (cudaStream_t)stream;
  const nfi::Plan r = nfi::route_backward(p, g);
  switch (r.route) {
    case nfi::Route::kRefused: return fail("%s", r.refusal);
    case nfi::Route::kSimt: return nfi::launch_backward_simt<false>(p, g, st);
    case nfi::Route::kSimtVd: return nfi::launch_backward_simt<true>(p, g, st);
    default: break;
  }
  unsigned char* ws = (unsigned char*)p.workspace;
  unsigned grid = 0;  // <= kMaxPersistentCtas: the accumulator rows are sized for that many CTAs
  if (int rc = persistent_grid(p, &grid)) return rc;
  if (r.route == nfi::Route::kPipeVd)
    return nfi::launch_pipe_backward<true>(p, g, ws, grid, st);
  if (r.route == nfi::Route::kPipe || r.route == nfi::Route::kPipeAndWgrad) {
    nfi_render_grads g1 = g;  // the decoder gradients are render_wgrad_pipe's
    g1.grad_w1 = g1.grad_b1 = g1.grad_w2 = g1.grad_b2 = nullptr;
    if (int rc = nfi::launch_pipe_backward<false>(p, g1, ws, grid, st)) return rc;
    if (r.route == nfi::Route::kPipe) return 0;
  }
  return nfi::launch_pipe_wgrad(p, g, ws, grid, r.route == nfi::Route::kWgradOneSweep, st);
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
      return fail("host entry point set-up failed: %s", cudaGetErrorString(e0)), 2;
    }
  }

  nfi_render_params d = *hp;
  const size_t B = hp->batch, H = hp->height, W = hp->width, S = hp->num_samples;
  const size_t R = hp->plane_res, A = hp->n_attention;
  const size_t nout = nfi::nout_of(hp->n_attention);
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
  // chunk = 8 images, ~34 MB per image on the wire
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
    fail("render failed: %s", cudaGetErrorString(e));
    rc = 2;
  }
  return rc;
}

}  // extern "C"
