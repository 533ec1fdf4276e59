/*
 * nfi_render.h -- C ABI of the H100 (sm_90a) fused tri-plane volume renderer.
 *
 * Drop-in boundary for ONE hot path of google-research/nerf-from-image: the
 * per-ray render (SURVEY.md section 8).  The reference has no FFI of its own
 * (it is 100 % Python/PyTorch); the seam it offers is the Python call
 *     render(target_model, height, width, tform_cam2world, focal_length,
 *            center, bbox, model_input, depth_samples_per_ray, ...)
 * at /root/reference/run.py:176-191, reached only from
 * ParallelModel.forward (run.py:597-611).  The entry points below are what a
 * ctypes binding of that seam calls; nerf_from_image_b200/render.py is that
 * binding and INTEGRATION.md shows the reference-side stub.
 *
 * Conventions
 *   - plain C types only; every pointer in nfi_render_params /
 *     nfi_render_grads is a DEVICE pointer to fp32 data owned by the caller
 *     (the *_host entry points take HOST pointers instead and do the copies);
 *   - `stream` is a cudaStream_t passed as void*; kernels are only enqueued,
 *     never synchronised (the *_host entry points synchronise before return);
 *   - the library keeps no mutable global state and is re-entrant: the
 *     reference's nn.DataParallel calls render() from one Python thread per
 *     GPU (run.py:636-644), and ctypes drops the GIL around each call;
 *   - return value 0 = success; anything else is an error whose text
 *     nfi_last_error() returns (thread-local).  The Python binding turns it
 *     into an exception, matching the reference's assert/raise behaviour
 *     (models/generator.py:412-421).
 */
#ifndef NFI_RENDER_H_
#define NFI_RENDER_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NFI_ABI_VERSION 6

#if defined(__GNUC__)
#define NFI_API __attribute__((visibility("default")))
#else
#define NFI_API
#endif

#define NFI_PLANE_CHANNELS 32 /* TriplanarDecoder(32, .)  models/generator.py:383 */
#define NFI_HIDDEN 64         /* hidden_dim             models/generator.py:293 */
#define NFI_MAX_ATTENTION 15  /* decoder outputs 1+A, padded to <= 16 */
#define NFI_MAX_PEERS 7       /* other GPUs of one NVSwitch domain */
#define NFI_VIEW_FEATURES 32  /* ViewDirectionMapper(., num_features=32) models/generator.py:191 */

/* what the 5th output of render() carries (run.py:227-257,337-338) */
enum nfi_extra_mode {
  NFI_EXTRA_NONE = 0,
  NFI_EXTRA_COORDS = 1,    /* compute_coords:    sum_i w_i * x_i      [B,H,W,3] */
  NFI_EXTRA_SEMANTICS = 2  /* compute_semantics: sum_i w_i * probs_i  [B,H,W,A] */
};

/* where the two random draws of the path come from */
enum nfi_noise_mode {
  NFI_NOISE_DETERMINISTIC = 0, /* randomize=False: no jitter, u = linspace(0,1,S) */
  NFI_NOISE_EXPLICIT = 1,      /* noise_t / noise_u tensors (torch.rand_like at
                                  lib/nerf_utils.py:112, torch.rand at :201) */
  NFI_NOISE_PHILOX = 2         /* nfi_render_forward_host only: both draws are generated ON THE
                                  DEVICE from noise_seed (Philox-4x32-10, as nfi_fill_uniform
                                  with stream ids 0 / 1) -- where the reference draws them
                                  too -- instead of crossing PCIe */
};

/* which implementation of the decoder MLP the kernels use */
enum nfi_mlp_mode {
  NFI_MLP_AUTO = 0,
  NFI_MLP_FP32_SIMT = 1, /* fp32 FFMA on CUDA cores                      */
  NFI_MLP_TC_3XTF32 = 2, /* alias of NFI_MLP_TC_PIPE (the lockstep tensor-core kernel, whose
                            tile groups gathered, decoded and shaded in turn, was retired) */
  NFI_MLP_TC_WARPSPEC = 3, /* alias of NFI_MLP_TC_PIPE (the first warp-specialised kernel, whose two
                              roles shared one ring stage per chain, was retired) */
  NFI_MLP_TC_PIPE = 4 /* same arithmetic, fully pipelined: A stages released at MMA completion,
                         hidden activations stay in registers, consumers software-pipelined
                         (default) */
};

typedef struct nfi_render_params {
  /* ---- shapes ---- */
  int32_t batch;       /* B */
  int32_t height;      /* H  (render(height, ...)) */
  int32_t width;       /* W */
  int32_t num_samples; /* S = depth_samples_per_ray: S coarse (+ S fine) */
  int32_t plane_res;   /* R: planes are [B,3,R,R,32] channel-last */
  int32_t n_attention; /* A: palette entries (args.attention_values); 0 = the
                          decoder emits 3 colour logits -> wide sigmoid */
  /* ---- flags (dataset_config / args read by render(), run.py:200-348) ---- */
  float scene_range;
  int32_t white_background;
  int32_t use_sdf;       /* 1: Laplace-CDF density, 0: softplus(d-1) */
  int32_t fine_sampling; /* args.fine_sampling: hierarchical pass on/off */
  int32_t noise_mode;    /* enum nfi_noise_mode */
  int32_t extra_mode;    /* enum nfi_extra_mode */
  int32_t compute_normals; /* analytic grad of the SDF, normalised, composited
                              with detached weights (generator.py:614-623): a second
                              pipelined kernel after the render (render_normals_pipe) */
  int32_t mlp_mode;      /* enum nfi_mlp_mode */
  /* ---- radiance field (models/generator.py:288-331,587-681) ---- */
  const float *planes; /* [B,3,R,R,32] channel-last, see nfi_planes_to_channel_last */
  const float *w1;     /* [64,32]  EFFECTIVE weight (EqualizedLinear gain applied) */
  const float *b1;     /* [64] */
  const float *w2;     /* [1+A,64] (or [4,64] when A == 0) */
  const float *b2;     /* [1+A] */
  const float *palette; /* [B,A,3] attention values, NULL when A == 0 */
  const float *beta;    /* [1] Generator.beta  (device scalar; NULL if !use_sdf) */
  const float *alpha;   /* [1] Generator.alpha */
  /* ---- cameras (lib/nerf_utils.py:28-91) ---- */
  const float *c2w;    /* [B,4,4] tform_cam2world */
  const float *focal;  /* [B] or NULL = orthographic model */
  const float *center; /* [B,2] or NULL */
  const float *bbox;   /* [B,2,2] (row 0 start, row 1 range) or NULL */
  /* ---- noise (NFI_NOISE_EXPLICIT) ---- */
  const float *noise_t; /* [B,H,W,S] in [0,1) */
  const float *noise_u; /* [B*H*W,S] in [0,1); only read when fine_sampling */
  /* ---- outputs ---- */
  float *rgb;     /* [B,H,W,3] */
  float *depth;   /* [B,H,W]   */
  float *mask;    /* [B,H,W]   */
  float *extra;   /* [B,H,W,3] or [B,H,W,A] or NULL (extra_mode) */
  float *normals; /* [B,H,W,3] or NULL */
  float *z_fine;  /* [B*H*W,S] sorted fine depths, kept for the backward pass and read by the
                     pipelined normals kernel (compute_normals without it: fp32 SIMT kernel);
                     NULL = do not save */
  /* ---- scratch ---- */
  void *workspace;        /* >= nfi_render_workspace_bytes(params) */
  size_t workspace_bytes;
  uint64_t noise_seed;    /* NFI_NOISE_PHILOX */
  /* ---- multi-GPU exchange fused into the render (ABI 4; nfi_render_forward, pipelined kernel) ----
   * The render's last step in the reference's multi-GPU form is the gather of every replica's
   * rgb / depth / mask tiles (nn.DataParallel, run.py:636-644).  With n_peers > 0 the kernel
   * stores each ray's outputs not only to rgb / depth / mask above but also, through NVLink peer
   * mappings, to the same ray of peer_*[q] for q < n_peers: THIS rank's slice inside peer q's
   * full-batch buffers (symmetric memory).  No collective call remains. */
  int32_t n_peers;        /* 0 .. NFI_MAX_PEERS */
  int32_t peer_reserved;
  float *peer_rgb[7];     /* [B,H,W,3] slices in the peers' address spaces */
  float *peer_depth[7];   /* [B,H,W] */
  float *peer_mask[7];    /* [B,H,W] */
  /* Optional completion handshake inside the kernel (peer_done != NULL): the LAST CTA of the
   * grid, after every CTA's stores are fenced system-wide, writes peer_epoch to peer_signal[q]
   * (a word in peer q's memory reserved for this rank) and waits until the words the peers
   * reserve for us here, peer_signal_self[peer_rank[q]], have reached peer_epoch.  When the
   * kernel has completed on a rank, all ranks' tiles are in its buffers: no barrier launch. */
  uint32_t *peer_signal[7];
  const uint32_t *peer_signal_self;
  int32_t peer_rank[7];
  uint32_t peer_epoch;
  uint32_t *peer_done;    /* zero-initialised device word (CTA counter), reset by the kernel */
  /* ---- view-direction conditioning (ABI 5; --use_viewdir, CARLA: run.py:216-217,
   * models/generator.py:189-253,376-377,662-663).  With view_features != NULL the decoder's
   * second layer emits 1 + 32 values (w2 [33,64], b2 [33]) and every sample's colour logits are
   *     w3 . leaky_relu(view_features[ray] + decoder_features, 0.2) + b3
   * (ViewDirectionMapper.mapper_closure); view_features is the mapper's per-RAY trunk output
   * (fc0 .. fc6 on the unit ray direction, computed by the caller once per ray).  Forward: the
   * pipelined tensor-core kernel inside its envelope (the fp32 SIMT kernel outside it or with
   * NFI_MLP_FP32_SIMT); backward: the pipelined tensor-core kernel with a frozen decoder and mapper
 * output inside its envelope (nfi_render_backward), the fp32 SIMT kernel otherwise. */
  const float *view_features; /* [B,H,W,32] or NULL */
  const float *w3;            /* [A,32] ([3,32] when A == 0): EFFECTIVE weight of mapper.output */
  const float *b3;            /* [A] ([3]) */
  /* ---- row tile (ABI 5): render rows [row_offset, row_offset + height) of images that are
   * full_height rows tall (full_height == 0: the whole image, height rows).  Every buffer of
   * this struct then has `height` rows; only the pixel -> ray mapping (lib/nerf_utils.py:36-39)
   * sees the offset.  This is how one image's rays are split over GPUs when there are fewer
   * images than GPUs (SURVEY.md section 8e; parallel.render_row_sharded). */
  int32_t row_offset;
  int32_t full_height;
} nfi_render_params;

/* Upstream gradients in, parameter gradients out (all device pointers).
 * Every grad_* output is ACCUMULATED into (+=); the caller zero-fills.  A NULL
 * output pointer skips that gradient (e.g. frozen decoder weights during
 * inversion, run.py:628-629 `model_ema.requires_grad_(False)`). */
typedef struct nfi_render_grads {
  const float *g_rgb;   /* [B,H,W,3] dL/d rgb */
  const float *g_mask;  /* [B,H,W] or NULL */
  const float *g_extra; /* like `extra` or NULL */
  const float *out_rgb;  /* forward outputs, needed for the suffix sums */
  const float *out_mask;
  const float *out_extra;
  float *grad_planes;  /* [B,3,R,R,32] channel-last */
  float *grad_w1;      /* [64,32] */
  float *grad_b1;      /* [64] */
  float *grad_w2;      /* [1+A,64] */
  float *grad_b2;      /* [1+A] */
  float *grad_palette; /* [B,A,3] */
  float *grad_beta;    /* [1] */
  float *grad_alpha;   /* [1] */
  float *grad_origins; /* [B,H,W,3] dL/d ray origin       (chain to c2w in the binding) */
  float *grad_dirs;    /* [B,H,W,3] dL/d unit ray direction */
  /* view-direction conditioning (ABI 5); grad_w2 / grad_b2 are then [33,64] / [33] */
  float *grad_view_features; /* [B,H,W,32] (overwritten per ray, not accumulated) */
  float *grad_w3;            /* [A,32] */
  float *grad_b3;            /* [A] */
} nfi_render_grads;

/* library / build identification */
NFI_API int nfi_abi_version(void);
NFI_API const char *nfi_build_info(void); /* "sm_90a ..." */
NFI_API const char *nfi_last_error(void);

/* Scratch the forward / backward kernels need for `params` (bytes). */
NFI_API size_t nfi_render_workspace_bytes(const nfi_render_params *params);

/* Planes arrive from SynthesisNetwork as [B,96,R,R] = three [B,32,R,R]
 * channel-first planes xy/xz/yz (models/generator.py:475-477,500-502).  The
 * render kernels gather channel-last texels (one 128-byte line per tap).
 * `batch_stride` is the element stride between images of each source plane. */
NFI_API int nfi_planes_to_channel_last(const float *xy, const float *xz, const float *yz,
                               int64_t batch_stride, int32_t batch, int32_t plane_res,
                               float *dst, void *stream);
/* inverse re-layout for the plane gradient: [B,3,R,R,32] -> [B,3,32,R,R] */
NFI_API int nfi_planes_from_channel_last(const float *src, int32_t batch, int32_t plane_res,
                                 float *dst, void *stream);

/* render() forward: run.py:176-350 from the planes on (rays, near/far, coarse
 * samples, field, importance resampling, sorted merge, compositing). */
NFI_API int nfi_render_forward(const nfi_render_params *params, void *stream);

/* TriplanarDecoder.net on given features (models/generator.py:294-299,329-331):
 * features [N,32] -> [N,1+A] (density-or-distance first, colour logits after).
 * Any mode but NFI_MLP_FP32_SIMT runs a 3xTF32 wgmma decoder tile (four 128-point
 * tiles per 512-thread CTA, weights split into TF32 hi / lo parts);
 * `workspace` must hold 32 KiB (ignored in SIMT mode). */
NFI_API int nfi_decoder_forward(const float *features, int64_t n_points, const float *w1,
                                const float *b1, const float *w2, const float *b2,
                                int32_t n_attention, float *out, int32_t mlp_mode,
                                void *workspace, void *stream);

/* autograd of the above (SURVEY.md section 8 row a13): recomputes the samples.
 * With params->workspace >= 64 KiB, no semantics output and S <= 128, S % 4 == 0 the four GEMMs of
 * a sample step run on the tensor cores (render_backward_pipe).  Decoder-weight gradients (grad_w1 /
 * b1 / w2 / b2) come from render_wgrad_pipe (MN-major bf16-pair GEMMs on wgmma), which needs
 * params->workspace >= NFI_BACKWARD_WORKSPACE_BYTES: without pose gradients (the GAN generator
 * step) it is the WHOLE backward in one sweep, with them it runs beside render_backward_pipe.
 * A view-conditioned render (params->view_features) takes the same envelope on its own
 * instantiation of render_backward_pipe when no grad_w1 / b1 / w2 / b2 / w3 / b3 is requested (the
 * inversion step: decoder and mapper frozen) and params->workspace holds
 * NFI_VIEW_BACKWARD_WORKSPACE_BYTES (its two weight images); grad_view_features may be NULL.
 * Everything outside that envelope: the fp32 SIMT kernel. */
#define NFI_BACKWARD_WORKSPACE_BYTES (65536 + 160 * 32768)
#define NFI_VIEW_BACKWARD_WORKSPACE_BYTES 98304
NFI_API int nfi_render_backward(const nfi_render_params *params, const nfi_render_grads *grads,
                        void *stream);

/* dst[i] = uniform in [0, 1) (24-bit, like torch.rand) from Philox-4x32-10 keyed by `seed`,
 * counter (offset + i) / 4, sub-stream `stream_id`; i in [0, n), offset % 4 == 0.  The value
 * of element `offset + i` does not depend on how a buffer is split into calls. */
NFI_API int nfi_fill_uniform(float *dst, int64_t n, uint64_t seed, uint32_t stream_id,
                             int64_t offset, void *stream);

/* Same as nfi_render_forward but every pointer in `params` (inputs and
 * outputs; `workspace` ignored) is a HOST pointer; `planes` is the
 * channel-FIRST [B,3,32,R,R] array the reference produces.  Copies in, runs,
 * copies rgb/depth/mask/extra/normals out and synchronises.  This is the
 * end-to-end entry the bench's `e2e` figure is measured through. */
NFI_API int nfi_render_forward_host(const nfi_render_params *params, int32_t device);

/* ---- secondary seam: the generator's `sampler` closure (SURVEY.md section 8b, B2) ----
 * models/generator.py:587-681 evaluated at arbitrary points: x = points / scene_range,
 * tri-plane fetch, decoder, then whichever of the outputs below are non-NULL.  Forward only
 * (the regulariser heads that differentiate through the closure stay on the reference path).
 * fp32 SIMT arithmetic -- this seam serves point clouds (marching cubes, the 31^3 regulariser
 * grids, SDF pre-training targets), not the per-ray hot loop. */
typedef struct nfi_sample_params {
  int32_t batch;       /* B */
  int32_t plane_res;   /* R */
  int32_t n_attention; /* A (0: three colour logits -> wide sigmoid) */
  int32_t use_sdf;
  int32_t bbox_debug;  /* 1: sigma += 100 on the cube's edges (generator.py:640-657) */
  float scene_range;
  int64_t n_points;    /* N points per image */
  const float *planes; /* [B,3,R,R,32] channel-last */
  const float *w1; /* effective decoder weights, as nfi_render_params */
  const float *b1;
  const float *w2;
  const float *b2;
  const float *palette; /* [B,A,3] or NULL */
  const float *beta; /* device scalars (use_sdf) */
  const float *alpha;
  const float *points;  /* [B,N,3] world units (x_in) */
  float *sdf_distance;  /* [B,N]   decoder output 0 ('sdf_distance')   or NULL */
  float *sigma;         /* [B,N]   ('sigma')                            or NULL */
  float *rgb;           /* [B,N,3] ('rgb')                              or NULL */
  float *semantics;     /* [B,N,A] softmax probabilities ('semantics')  or NULL */
  float *normals;       /* [B,N,3] normalised grad of the SDF ('normals') or NULL */
} nfi_sample_params;
NFI_API int nfi_sample_field(const nfi_sample_params *params, void *stream);

/* ---- neighbour of the path in the inversion loop (SURVEY.md section 8f, N4) ----
 * lib/pose_utils.py:48-70 pose_to_matrix: (z0|NULL, t2 [B,2], s [B], q [B,4] unit quaternion)
 * -> tform_cam2world [B,4,4] (+ focal [B] = (1 + e^z0) / 2 when z0 is given; z0 == NULL is the
 * orthographic model: translation (t2, 10), whole matrix divided by s).  One thread per image. */
NFI_API int nfi_pose_to_matrix(const float *z0, const float *t2, const float *s, const float *q,
                               int32_t camera_flipped, int32_t batch, float *c2w, float *focal,
                               void *stream);
/* its vector-Jacobian product: g_c2w [B,4,4], g_focal [B]|NULL in; g_z0 (NULL iff z0 NULL),
 * g_t2, g_s, g_q out (overwritten). */
NFI_API int nfi_pose_to_matrix_backward(const float *z0, const float *t2, const float *s,
                                        const float *q, int32_t camera_flipped, int32_t batch,
                                        const float *g_c2w, const float *g_focal, float *g_z0,
                                        float *g_t2, float *g_s, float *g_q, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NFI_RENDER_H_ */
