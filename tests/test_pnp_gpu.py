"""The PnP kernels (nfi_pnp.cu) against the float64 oracle and the recorded OpenCV outputs, on the
GPU; no cv2 or reference needed."""
import numpy as np
import pytest
import torch

from nerf_from_image_b200 import pnp
from nerf_from_image_b200._lib import NfiError
from oracle import pnp_oracle as O
from tests import pnp_cases as C
from tests.test_pnp_oracle import CASES, GOLDEN, DISAGREEMENTS, compare

pytestmark = pytest.mark.gpu


def run(coords, mask, focals, refine=True):
    co = torch.from_numpy(np.ascontiguousarray(coords)).cuda()
    m = torch.from_numpy(np.ascontiguousarray(mask)).cuda()
    w, f, e = pnp.compute_pose_pnp(co, m, focals, refine=refine)
    rec = pnp.candidate_records(co, m, focals, refine=refine)
    return (w.cpu().numpy(), f.cpu().numpy(), e.cpu().numpy()), rec.cpu().numpy()


@pytest.mark.parametrize('name', sorted(CASES))
def test_kernels_match_the_oracle(name, cuda_lib):
    co, m, f, refine = CASES[name]
    (w, fo, e), rec = run(co, m, f, refine)
    recs = []
    ow, ofo, oe = O.compute_pose_pnp(co, m, f, refine=refine, records=recs)
    assert np.array_equal(fo, ofo), (fo, ofo)
    for b, r in enumerate(recs):
        assert [c['solver'] for c in r] == list(rec[b, :len(r), 0].astype(int))
        assert [int(c['accepted']) for c in r] == list(rec[b, :len(r), 1].astype(int))
    assert np.max(np.abs(w - ow)) <= 1e-9, np.max(np.abs(w - ow))
    assert np.max(np.abs(e - oe) / np.abs(oe)) <= 1e-9


@pytest.mark.parametrize('name', sorted(CASES))
def test_kernels_match_the_recorded_reference(name, cuda_lib):
    co, m, f, refine = CASES[name]
    got, _ = run(co, m, f, refine)
    g = np.load('%s/pnp_%s.npz' % (GOLDEN, name))
    assert compare(got, (g['world2cam'], g['focal'], g['error']), name) <= DISAGREEMENTS.get(name, 0)


def test_orthographic_estimate_poses_batch(cuda_lib):
    co, m, _, _ = CASES['orthographic']
    c2w, focal, _ = pnp.estimate_poses_batch(torch.from_numpy(co).cuda(),
                                             torch.from_numpy(m.astype(np.float32)).cuda(), None)
    assert focal is None and c2w.dtype == torch.float32 and c2w.is_cuda
    g = np.load('%s/pnp_orthographic.npz' % GOLDEN)
    w = g['world2cam'].copy()   # run.py's conversion of the recorded reference output
    s = 2 * 100. / -w[:, 2, 3]
    w[:, :2, 3] *= s[:, None]
    w[:, 2, 3] = -10.
    want = pnp.invert_space(torch.from_numpy(w).float()) / torch.from_numpy(s[:, None, None]).float()
    assert torch.allclose(c2w.cpu(), want, rtol=1e-5, atol=1e-5)


def test_strided_encoder_view(cuda_lib):
    co, m, f, refine = CASES['perspective']
    maps = torch.zeros(co.shape[:3] + (4,), device='cuda')
    maps[..., :3] = torch.from_numpy(co).cuda()
    view = maps[..., :3]
    assert not view.is_contiguous()
    a = pnp.compute_pose_pnp(view, torch.from_numpy(m).cuda(), f)
    b = pnp.compute_pose_pnp(view.contiguous(), torch.from_numpy(m).cuda(), f)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize('batch', [1, 16, 64])
def test_sizes_recover_the_cameras(batch, cuda_lib):
    co, m, w2c = C.ellipsoid_views(batch, batch, res=128, focal=2.0)
    w, fo, e = pnp.compute_pose_pnp(torch.from_numpy(co).cuda(), torch.from_numpy(m).cuda(),
                                    C.FOCAL_GUESSES)
    flip = torch.diag(torch.tensor([1., -1., -1., 1.], dtype=torch.float64))
    truth = flip @ torch.from_numpy(w2c)
    assert torch.all(fo.cpu() == 2.0)
    assert (w.cpu() - truth).abs().max() < 2e-2
    assert torch.all(e.cpu() < 5e-3)


def test_bit_identical_alone_in_a_batch_and_across_calls(cuda_lib):
    co, m, _ = C.ellipsoid_views(5, 16, res=128, focal=2.0)
    cot, mt = torch.from_numpy(co).cuda(), torch.from_numpy(m).cuda()
    a = pnp.compute_pose_pnp(cot, mt, C.FOCAL_GUESSES)
    b = pnp.compute_pose_pnp(cot, mt, C.FOCAL_GUESSES)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    one = pnp.compute_pose_pnp(cot[5:6], mt[5:6], C.FOCAL_GUESSES)
    assert all(torch.equal(x[5:6], y) for x, y in zip(a, one))


def test_refusals(cuda_lib):
    co, m, f, _ = CASES['perspective']
    cot, mt = torch.from_numpy(co), torch.from_numpy(m)
    with pytest.raises(NfiError):
        pnp.compute_pose_pnp(cot, mt, f)                                  # CPU
    with pytest.raises(NfiError):
        pnp.compute_pose_pnp(cot.cuda().double(), mt.cuda(), f)          # dtype
    with pytest.raises(NfiError):
        pnp.compute_pose_pnp(cot.cuda()[..., :2], mt.cuda(), f)          # shape
    with pytest.raises(NfiError):
        pnp.compute_pose_pnp(cot.cuda(), mt.cuda()[:, :-1], f)           # mask shape
    with pytest.raises(NfiError):
        pnp.compute_pose_pnp(cot.cuda(), mt.cuda(), [])                   # no guesses


@pytest.mark.parametrize('case', ['p3d_plain', 'cub_ortho'])
def test_render_round_trip(case, cuda_lib):
    """Coords and mask rendered by the fused render from the synthetic SDF scene at known cameras;
    estimate_poses_batch recovers the cameras.  The render composites sum_i w_i x_i, which is on
    the pixel's ray only where sum_i w_i = 1, so the points given to PnP are coords / mask (the
    expected surface point of the ray)."""
    from fixtures import synthetic
    from nerf_from_image_b200 import _lib
    from tests import helpers as Hh
    B, H, W, S = 4, 64, 64, 32
    scene, cams = Hh.make_case(case, batch=B, plane_res=64)
    scene['alpha'] = scene['alpha'] * 0.02   # a sharp surface: the mask reaches 1 on the object
    ortho = cams['focal'] is None
    if not ortho:
        cams['focal'] = torch.full((B,), 1.3)
    nt, nu = synthetic.make_noise(1, B, H, W, S)
    with torch.no_grad():
        _, _, mask, coords = Hh.run_cuda(scene, cams, H, W, S, nt, nu, extra_mode=_lib.EXTRA_COORDS,
                                         cam_grad=False)
    mask = mask.reshape(B, H, W)
    coords = coords.reshape(B, H, W, 3) / mask.clamp_min(1e-6)[..., None]
    assert torch.all((mask > 0.9).reshape(B, -1).sum(1) >= 50)
    guesses = None if ortho else [1.0, 1.1, 1.2, 1.3, 1.4, 1.5]
    c2w, focal, err = pnp.estimate_poses_batch(coords.contiguous(), mask, guesses)
    true = cams['c2w'].double()
    c2w = c2w.double().cpu()
    if not ortho:
        assert torch.all(focal.cpu() == 1.3)
        assert (c2w - true).abs().max() < 1e-3, (c2w - true).abs().max()
        assert torch.all(err.cpu() < 1e-4)
    else:
        # orthographic: focal 100 stands in for the parallel projection (depth is not observable;
        # run.py puts the camera at 10 / s along its axis), so compare the rotation, the scale and
        # the camera's offset across its axis.  The render's orthographic rays start on a plane 2
        # world units across whatever c2w[3,3] is (it scales only their direction), so the
        # footprint the estimate recovers is s = 1: c2w[3,3] = 1
        c33 = c2w[:, 3, 3]
        assert (c2w[:, :3, :3] / c33[:, None, None] - true[:, :3, :3]).abs().max() < 5e-3
        assert (c33 - 1).abs().max() < 5e-3, c33
        o = c2w[:, :3, 3] / c33[:, None]
        axis = true[:, :3, 2]
        across = o - (o * axis).sum(1, keepdim=True) * axis
        assert across.abs().max() < 5e-3, across.abs().max()
