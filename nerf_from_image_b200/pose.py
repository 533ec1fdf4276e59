"""``pose_to_matrix`` of the inversion loop as one kernel each way (SURVEY.md 8f, N4).

Same call as ``lib/pose_utils.py:48-70``: ``pose_to_matrix(z0, t2, s, q,
camera_flipped) -> (tform_cam2world [B,4,4], focal [B] | None)``; ``z0 is
None`` selects the orthographic model.  The reference builds the matrix from
~25 elementwise / indexing launches and autograd replays about twice that on
the way back, every optimisation step (run.py:2202-2254); here the forward and
the vector-Jacobian product are one launch each (``nfi_pose_to_matrix``,
``nfi_pose_to_matrix_backward``), and the result feeds ``render`` directly.
"""

import torch

from . import _lib


def _prep(t, name, shape_tail):
    if t is None:
        return None
    if not t.is_cuda:
        raise _lib.NfiError('%s must be a CUDA tensor: pose_to_matrix has no CPU path' % name)
    if tuple(t.shape[1:]) != shape_tail:
        raise _lib.NfiError('%s must be [B%s]' % (name, ''.join(',%d' % d for d in shape_tail)))
    return t.detach().to(torch.float32).contiguous()


class PoseToMatrix(torch.autograd.Function):

    @staticmethod
    def forward(ctx, z0, t2, s, q, camera_flipped):
        q_ = _prep(q, 'q', (4,))
        B = q_.shape[0]
        z0_, t2_, s_ = _prep(z0, 'z0', ()), _prep(t2, 't2', (2,)), _prep(s, 's', ())
        if t2_.shape[0] != B or s_.shape[0] != B or (z0_ is not None and z0_.shape[0] != B):
            raise _lib.NfiError('z0 / t2 / s / q disagree on the batch size')
        mat = torch.empty(B, 4, 4, device=q_.device, dtype=torch.float32)
        focal = torch.empty(B, device=q_.device, dtype=torch.float32) if z0_ is not None else None
        lib = _lib.load()
        with torch.cuda.device(q_.device):
            stream = _lib.stream(q_.device)
            _lib.check(lib.nfi_pose_to_matrix(_lib.ptr(z0_), _lib.ptr(t2_), _lib.ptr(s_), _lib.ptr(q_),
                                              int(bool(camera_flipped)), B, _lib.ptr(mat),
                                              _lib.ptr(focal), stream))
        ctx.save_for_backward(*(t for t in (z0_, t2_, s_, q_) if t is not None))
        ctx.persp = z0_ is not None
        ctx.flipped = int(bool(camera_flipped))
        return mat, focal

    @staticmethod
    def backward(ctx, g_mat, g_focal):
        if ctx.persp:
            z0, t2, s, q = ctx.saved_tensors
        else:
            (t2, s, q), z0 = ctx.saved_tensors, None
        B = q.shape[0]
        g_mat = (g_mat if g_mat is not None else torch.zeros(B, 4, 4, device=q.device)) \
            .to(torch.float32).contiguous()
        g_focal = g_focal.to(torch.float32).contiguous() if (ctx.persp and g_focal is not None) \
            else None
        g_z0 = torch.empty_like(z0) if ctx.persp else None
        g_t2, g_s, g_q = torch.empty_like(t2), torch.empty_like(s), torch.empty_like(q)
        lib = _lib.load()
        with torch.cuda.device(q.device):
            stream = _lib.stream(q.device)
            _lib.check(lib.nfi_pose_to_matrix_backward(
                _lib.ptr(z0), _lib.ptr(t2), _lib.ptr(s), _lib.ptr(q), ctx.flipped, B, _lib.ptr(g_mat),
                _lib.ptr(g_focal), _lib.ptr(g_z0), _lib.ptr(g_t2), _lib.ptr(g_s), _lib.ptr(g_q),
                stream))
        return g_z0, g_t2, g_s, g_q, None


def pose_to_matrix(z0, t2, s, q, camera_flipped: bool):
    """lib/pose_utils.py:48-70.  Returns (mat, focal) -- focal is None when z0 is."""
    return PoseToMatrix.apply(z0, t2, s, q, camera_flipped)
