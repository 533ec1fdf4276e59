"""Install the reference's PnP pose initialisation for the comparisons -- TEST / BASELINE
INFRASTRUCTURE.

Copies lib/pose_estimation.py UNMODIFIED from a checkout of google-research/nerf-from-image into
the same git-ignored ``oracle/_ref/`` that ``oracle/stage_reference.py`` fills.  It imports cv2,
numpy and torch; where cv2 is importable, tests/test_pnp_oracle.py runs its compute_pose_pnp live
against oracle/pnp_oracle.py, and tools/time_pnp.py times it.  Elsewhere the comparisons use the
outputs recorded under tests/golden/reference/.
"""
import hashlib
import json
import os
import shutil
import sys

try:
    from oracle import stage_reference
except ImportError:   # run as a script: oracle/ is on the path, the repository root is not
    import stage_reference

FILES = ('lib/pose_estimation.py',)


def stage(src=stage_reference.SRC, dest=stage_reference.DEST, quiet=False):
    """Copies FILES from ``src`` to ``dest``; returns the manifest (path -> sha256)."""
    if not available(src):
        raise FileNotFoundError('no reference pose estimation at %s' % src)
    manifest = {}
    for rel in FILES:
        s, d = os.path.join(src, rel), os.path.join(dest, rel)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        shutil.copyfile(s, d)
        with open(d, 'rb') as f:
            manifest[rel] = hashlib.sha256(f.read()).hexdigest()
    with open(os.path.join(dest, 'MANIFEST.pnp.json'), 'w') as f:
        json.dump({'source': src, 'files': manifest}, f, indent=1, sort_keys=True)
    if not quiet:
        print('staged %d reference PnP file into %s' % (len(manifest), dest))
    return manifest


def available(root):
    """Whether ``root`` (a staged or checked-out reference) has the file."""
    return all(os.path.isfile(os.path.join(root, rel)) for rel in FILES)


def reference_compute_pose_pnp():
    """The staged reference's compute_pose_pnp, or None without the staged file or cv2."""
    path = os.path.join(stage_reference.DEST, FILES[0])
    if not os.path.isfile(path):
        return None
    try:
        import cv2  # noqa: F401
    except ImportError:
        return None
    import importlib.util
    spec = importlib.util.spec_from_file_location('_nfi_ref_pose_estimation', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.compute_pose_pnp


if __name__ == '__main__':
    stage(*(sys.argv[1:2] or [stage_reference.SRC]))
