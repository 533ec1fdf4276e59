/*
 * nfi_pnp.h -- C ABI of the inversion's pose initialisation: batched PnP from the bootstrap
 * encoder's canonical coordinate maps (README design 4.12).
 *
 * For each image b and each focal guess f (in order) the library solves the perspective-n-point
 * problem of its foreground pixels (mask != 0, row-major pixel order): 3D point coords[b, y, x]
 * in float64, screen point (x/W - 0.5, y/H - 0.5), intrinsics fx = fy = focal, principal point 0.
 * SQPnP first; EPnP when SQPnP has no solution with t_z > 0; then, with refine, Levenberg-Marquardt
 * on (Rodrigues rvec, t), kept when its t_z > 0.  The error is the RMS reprojection error
 * sqrt(sum |proj - screen|^2 / (2N)).  Per image the guess with the strictly smallest error wins;
 * with no pose (fewer than 4 points, or no guess solved) the image gets rvec 0, t = (0, 0, -10),
 * focal 1, error 10.  world2cam = diag(1, -1, -1, 1) [R(rvec) | t].
 *
 * All in float64, no atomics: an image's result is the same bits alone and in any batch.
 * Conventions as in nfi_render.h: device pointers, stream as void*, 0 = success.
 */
#ifndef NFI_PNP_H_
#define NFI_PNP_H_

#include <stddef.h>
#include <stdint.h>

#include "nfi_render.h"

#ifdef __cplusplus
extern "C" {
#endif

#define NFI_PNP_MAX_FOCALS 64
/* one candidate record: solver (0 none, 1 SQPnP, 2 EPnP), refinement accepted (0/1), rvec[3],
   t[3], error -- all stored as double */
#define NFI_PNP_RECORD_DOUBLES 9

typedef struct nfi_pnp_params {
  int32_t batch;              /* B */
  int32_t height;             /* H */
  int32_t width;              /* W */
  int32_t n_focals;           /* F, 1..NFI_PNP_MAX_FOCALS */
  int32_t refine;             /* 0 / 1 */
  const float *coords;        /* [B,H,W,3] fp32 at the strides below (a strided view is fine) */
  int64_t coords_stride[4];   /* element strides of b, y, x, channel */
  const uint8_t *mask;        /* [B,H,W] contiguous, nonzero = foreground */
  const double *focals;       /* [F] */
  double *world2cam;          /* out [B,4,4] */
  double *focal;              /* out [B] */
  double *error;              /* out [B] */
  double *record;             /* out [B,F,NFI_PNP_RECORD_DOUBLES] per candidate, or NULL */
  void *workspace;
  size_t workspace_bytes;
} nfi_pnp_params;

/* bytes of workspace nfi_pnp_solve needs; 0 (reason in nfi_last_error) for a refused shape */
NFI_API size_t nfi_pnp_workspace_bytes(const nfi_pnp_params *params);
NFI_API int nfi_pnp_solve(const nfi_pnp_params *params, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NFI_PNP_H_ */
