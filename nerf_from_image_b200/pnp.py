"""The inversion's pose initialisation on the GPU (include/nfi_pnp.h, README design 4.12).

``compute_pose_pnp`` is the reference's lib/pose_estimation.py function on CUDA tensors, and
``estimate_poses_batch`` is run.py's, with the cameras left on the device: no host copy, no sync.
There is no fallback: CPU tensors, wrong shapes or dtypes raise ``NfiError``.
"""
import ctypes

import torch

from . import _lib
from ._lib import NfiError

SOLVER_NONE, SOLVER_SQPNP, SOLVER_EPNP = 0, 1, 2


def _solve(coords, masks, focals, refine, record):
    if not (torch.is_tensor(coords) and torch.is_tensor(masks)):
        raise NfiError('pnp: coords and masks must be tensors')
    if not coords.is_cuda or masks.device != coords.device:
        raise NfiError('pnp: coords and masks must be CUDA tensors on one device')
    if coords.dtype != torch.float32 or coords.dim() != 4 or coords.shape[-1] != 3:
        raise NfiError('pnp: coords must be float32 [B,H,W,3], got %s %s'
                       % (coords.dtype, tuple(coords.shape)))
    B, H, W, _ = coords.shape
    if masks.shape != (B, H, W) or masks.dtype not in (torch.bool, torch.uint8):
        raise NfiError('pnp: masks must be bool or uint8 [B,H,W] = %s, got %s %s'
                       % ((B, H, W), masks.dtype, tuple(masks.shape)))
    if torch.is_tensor(focals):
        focals = focals.detach().to(coords.device, torch.float64).reshape(-1).contiguous()
    else:
        focals = torch.tensor([float(f) for f in focals], dtype=torch.float64, device=coords.device)
    F = focals.numel()
    dev = coords.device
    mask_u8 = masks.contiguous().view(torch.uint8) if masks.dtype == torch.bool else masks.contiguous()
    world2cam = torch.empty(B, 4, 4, dtype=torch.float64, device=dev)
    focal = torch.empty(B, dtype=torch.float64, device=dev)
    error = torch.empty(B, dtype=torch.float64, device=dev)
    rec = torch.empty(B, max(F, 1), _lib.PNP_RECORD_DOUBLES, dtype=torch.float64, device=dev) \
        if record else None
    p = _lib.PnpParams()
    p.batch, p.height, p.width, p.n_focals, p.refine = B, H, W, F, int(bool(refine))
    p.coords = _lib.ptr(coords)
    p.coords_stride[:] = list(coords.stride())
    p.mask, p.focals = _lib.ptr(mask_u8), _lib.ptr(focals)
    p.world2cam, p.focal, p.error, p.record = (_lib.ptr(world2cam), _lib.ptr(focal), _lib.ptr(error),
                                               _lib.ptr(rec))
    lib = _lib.load()
    need = lib.nfi_pnp_workspace_bytes(ctypes.byref(p))
    if need == 0:
        _lib.check(1)
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    p.workspace, p.workspace_bytes = _lib.ptr(ws), need
    with torch.cuda.device(dev):
        _lib.check(lib.nfi_pnp_solve(ctypes.byref(p), _lib.stream(dev)))
    return world2cam, focal, error, rec


def compute_pose_pnp(coords, masks, focal_proposals, refine=True):
    """(world2cam [B,4,4], focal [B], error [B]), float64 CUDA tensors: the reference's
    compute_pose_pnp for CUDA ``coords`` [B,H,W,3] float32 (a strided view such as the encoder's
    ``maps[..., :3]`` is read in place) and ``masks`` [B,H,W] bool."""
    return _solve(coords, masks, focal_proposals, refine, False)[:3]


def candidate_records(coords, masks, focal_proposals, refine=True):
    """The per-(image, focal) records [B,F,9]: solver (0 none, 1 SQPnP, 2 EPnP), refinement
    accepted, rvec[3], t[3], error.  For tests."""
    return _solve(coords, masks, focal_proposals, refine, True)[3]


def invert_space(mat):
    """cam2world <-> world2cam of [B,4,4] matrices with a scale in [3,3] (lib/pose_utils.py)."""
    out = torch.zeros_like(mat)
    out[:, :3, :3] = mat[:, :3, :3].transpose(-2, -1) / mat[:, 3:4, 3:4]
    out[:, 3, 3] = 1
    out[:, :3, 3] = -torch.sum(mat[:, :3, :3] / mat[:, 3:4, 3:4] * mat[:, :3, None, 3], dim=-2)
    return out


def estimate_poses_batch(target_coords, target_mask, focal_guesses):
    """run.py's estimate_poses_batch on the device: (cam2world [B,4,4] float32, focal [B] float32
    or None for the orthographic case, errors [B] float64), all CUDA tensors."""
    if not torch.is_tensor(target_mask) or not target_mask.is_floating_point():
        raise NfiError('pnp: target_mask must be a floating-point tensor')
    masks = target_mask > 0.9
    is_ortho = focal_guesses is None
    if is_ortho:
        focal_guesses = [100.]   # a large focal length approximates the orthographic projection
    world2cam, focal, errors = compute_pose_pnp(target_coords, masks, focal_guesses)
    if is_ortho:
        s = 2 * float(focal_guesses[0]) / -world2cam[:, 2, 3]
        world2cam = world2cam.clone()
        world2cam[:, :2, 3] = world2cam[:, :2, 3] * s[:, None]
        world2cam[:, 2, 3] = -10.
    cam2world = invert_space(world2cam.float())
    if is_ortho:
        cam2world = cam2world / s[:, None, None].float()
        return cam2world, None, errors
    return cam2world, focal.float(), errors
