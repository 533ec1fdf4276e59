"""Seeded inputs of the PnP pose initialisation (tests/test_pnp_*.py, tools/time_pnp.py).

Each case is (coords [B,H,W,3] float32, mask [B,H,W] bool, focal guesses or None): the canonical
coordinate map and mask the bootstrap encoder predicts, made here by casting each pixel's ray
at a known camera onto an ellipsoid and adding noise to the hit points.
"""
import numpy as np

FOCAL_GUESSES = [1.2, 1.35, 1.5, 1.65, 1.8, 2.0, 2.2, 2.4, 2.7, 3.0, 3.4]  # 11, as get_focal_guesses


def _rotation(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def ellipsoid_views(seed, batch, res=128, focal=2.0, noise=2e-3, ortho=False, radii=(0.45, 0.3, 0.35),
                    distance=2.6):
    """Views of an ellipsoid at random rotations: coords are the world hit points plus Gaussian
    noise.  ``ortho``: parallel rays (the orthographic datasets).  Also returns the true
    world2cam [B,4,4] (OpenCV convention: camera looks down +z)."""
    rng = np.random.default_rng(seed)
    radii = np.asarray(radii)
    u = (np.arange(res) / res) - 0.5
    sx, sy = np.meshgrid(u, u, indexing='xy')
    coords = np.zeros((batch, res, res, 3), np.float32)
    mask = np.zeros((batch, res, res), bool)
    w2c = np.zeros((batch, 4, 4))
    for b in range(batch):
        rot = _rotation(rng)
        t = np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.1, 0.1), distance])
        if ortho:
            o = np.stack([sx * 2.0, sy * 2.0, np.zeros_like(sx)], -1) - np.array([0, 0, 10.0])
            d = np.broadcast_to(np.array([0.0, 0.0, 1.0]), o.shape)
        else:
            o = np.zeros(sx.shape + (3,))
            d = np.stack([sx / focal, sy / focal, np.ones_like(sx)], -1)
        # into world space: X = R^T (Xc - t)
        ow = (o - t) @ rot
        dw = d @ rot
        a = np.sum((dw / radii) ** 2, -1)
        bb = 2 * np.sum(ow * dw / radii ** 2, -1)
        c = np.sum((ow / radii) ** 2, -1) - 1
        disc = bb * bb - 4 * a * c
        hit = disc > 0
        s = (-bb - np.sqrt(np.maximum(disc, 0))) / (2 * a)
        p = ow + s[..., None] * dw
        coords[b] = p + rng.normal(scale=noise, size=p.shape)
        mask[b] = hit
        w2c[b, :3, :3], w2c[b, :3, 3], w2c[b, 3, 3] = rot, t, 1
    return coords, mask, w2c


def random_coords(seed, batch, res=32, fill=0.5):
    """Coordinates with no geometry behind them: uniform noise in the unit cube on a random mask.
    SQPnP often finds no solution in front of the camera here and EPnP runs."""
    rng = np.random.default_rng(seed)
    coords = rng.uniform(-0.5, 0.5, size=(batch, res, res, 3)).astype(np.float32)
    mask = rng.uniform(size=(batch, res, res)) < fill
    return coords, mask


def few_points(counts, res=16, seed=0):
    """One image per entry of ``counts`` with exactly that many foreground pixels."""
    coords, mask, _ = ellipsoid_views(seed, len(counts), res=res, focal=2.0)
    out = np.zeros_like(mask)
    for b, n in enumerate(counts):
        idx = np.nonzero(mask[b].reshape(-1))[0]
        keep = idx[np.linspace(0, len(idx) - 1, n).astype(int)] if n else idx[:0]
        out[b].reshape(-1)[keep] = True
    return coords, out


def cases():
    """name -> (coords, mask, focal guesses, refine): the comparisons' inputs."""
    persp = ellipsoid_views(1, 4, res=64)
    ortho = ellipsoid_views(2, 4, res=64, ortho=True)
    norefine = ellipsoid_views(4, 3, res=64)
    few = few_points([0, 3, 4, 5])
    rnd = random_coords(3, 8)
    rej = random_coords(24, 4, res=16, fill=0.3)
    return {
        'perspective': (persp[0], persp[1], FOCAL_GUESSES, True),
        'orthographic': (ortho[0], ortho[1], [100.], True),
        'no_refine': (norefine[0], norefine[1], FOCAL_GUESSES, False),
        'few_points': (few[0], few[1], FOCAL_GUESSES[:3], True),
        'random': (rnd[0], rnd[1], FOCAL_GUESSES[:3], True),
        'rejected_refinement': (rej[0], rej[1], [1.2, 2.0], True),
    }


WELL_POSED = ('perspective', 'orthographic', 'no_refine')
