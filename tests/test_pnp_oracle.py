"""oracle/pnp_oracle.py against the reference's compute_pose_pnp (OpenCV): live where cv2 and the
staged reference are importable, otherwise against its outputs recorded under
tests/golden/reference/."""
import os

import numpy as np
import pytest

from oracle import pnp_oracle as O
from oracle import stage_pnp_reference
from tests import pnp_cases as C

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference')
CASES = C.cases()
# Images whose decisions differ from cv2 4.13, measured.  `rejected_refinement` (random coordinates,
# ~80 points): on images 1 and 3 OpenCV's SQPnP and this one return different minima of the same
# algebraic error, so different starts reach the LM.  `few_points`: the image of exactly four points,
# where M^T M has a four-dimensional null space and EPnP's basis of it is arbitrary.
DISAGREEMENTS = {'rejected_refinement': 2, 'few_points': 1}


def reference(name):
    co, m, f, refine = CASES[name]
    ref = stage_pnp_reference.reference_compute_pose_pnp()
    if ref is not None:
        w, fo, e = ref(co, m, f, refine=refine)
        return np.asarray(w), np.asarray(fo, np.float64), np.asarray(e, np.float64)
    g = np.load(os.path.join(GOLDEN, 'pnp_%s.npz' % name))
    return g['world2cam'], g['focal'], g['error']


def compare(got, want, name):
    """Raises unless ``got`` meets the agreement bars of ``name``'s kind against ``want``."""
    (w, fo, e), (rw, rfo, re_) = got, want
    if name in C.WELL_POSED:
        assert np.array_equal(fo, rfo), (fo, rfo)
        assert np.max(np.abs(w[:, :3, :3] - rw[:, :3, :3])) <= 1e-6
        assert np.all(np.linalg.norm(w[:, :3, 3] - rw[:, :3, 3], axis=1)
                      <= 1e-6 * np.linalg.norm(rw[:, :3, 3], axis=1))
        assert np.all(np.abs(e - re_) <= 1e-6 * np.abs(re_))
        return 0
    same = (fo == rfo) & ((e == 10.) == (re_ == 10.))
    both = same & (re_ != 10.)
    assert np.all(np.abs(e - re_)[both] <= 1e-6 * np.abs(re_)[both]) or not both.any()
    return int(np.sum(~same) + np.sum(both & (np.abs(e - re_) > 1e-6 * np.abs(re_))))


@pytest.mark.parametrize('name', sorted(CASES))
def test_oracle_matches_the_reference(name):
    co, m, f, refine = CASES[name]
    got = O.compute_pose_pnp(co, m, f, refine=refine)
    bad = compare(got, reference(name), name)
    assert bad <= DISAGREEMENTS.get(name, 0), bad


@pytest.mark.parametrize('name', sorted(CASES))
def test_epnp_matches_opencv(name):
    """EPnP alone against cv2.SOLVEPNP_EPNP on every (image, focal) of the fixtures with more than
    five points: rotation and t within 1e-6 (measured <= 3e-8)."""
    cv2 = pytest.importorskip('cv2')
    co, m, f, _ = CASES[name]
    for b in range(co.shape[0]):
        pts, scr = O.foreground(co[b], m[b])
        if len(pts) <= 5:
            continue
        for focal in f:
            k = np.diag([focal, focal, 1.0])
            _, rv, tv, _ = cv2.solvePnPGeneric(pts, scr, k, None, flags=cv2.SOLVEPNP_EPNP)
            r, t = O.epnp(pts, scr, focal)
            assert np.abs(r - cv2.Rodrigues(rv[0])[0]).max() <= 1e-6
            assert np.linalg.norm(t - tv[0].ravel()) <= 1e-6 * np.linalg.norm(tv[0])


def test_cases_take_every_path():
    """EPnP runs on random inputs, a refinement is rejected, and few points give the dummy pose."""
    recs = []
    co, m, f, refine = CASES['random']
    O.compute_pose_pnp(co, m, f, refine=refine, records=recs)
    assert any(c['solver'] == O.SOLVER_EPNP for r in recs for c in r)
    recs = []
    co, m, f, refine = CASES['rejected_refinement']
    O.compute_pose_pnp(co, m, f, refine=refine, records=recs)
    assert any(c['solver'] != O.SOLVER_NONE and not c['accepted'] for r in recs for c in r)
    recs = []
    co, m, f, refine = CASES['orthographic']
    O.compute_pose_pnp(co, m, f, refine=refine, records=recs)
    assert all(c['solver'] == O.SOLVER_EPNP for r in recs for c in r)   # too little image spread
    w, fo, e = O.compute_pose_pnp(*CASES['few_points'][:3])
    assert list(e[:2]) == [10., 10.] and list(fo[:2]) == [1., 1.] and np.all(e[2:] < 1)
