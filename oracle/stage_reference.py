"""Install the reference's hot-path sources for the comparisons -- TEST / BASELINE INFRASTRUCTURE.

The files the lifted reference needs (oracle/reference_lift.py: `render` out of run.py by AST,
the reference Generator, its synthesis network, nerf_utils, ops, pose_utils) are copied
UNMODIFIED from a checkout of google-research/nerf-from-image into `oracle/_ref/` --
git-ignored, never part of this repository's history.  The reference has no setup.py /
pyproject.toml, so `pip install --target oracle/_ref` is not possible and a file-level copy of
the Apache-2.0 sources is what "install" means here.

Used by: `__graft_entry__.build()` (when a checkout exists at $NFI_REFERENCE_SRC, default
/root/reference), then by `oracle/reference_lift.py` -> the tests that compare against the
reference running on the same machine, and `bench.py --impl reference`
(`cpu_baseline.kind == "reference"`).  Without it those comparisons fall back to the committed
golden vectors or skip.
"""
import hashlib
import json
import os
import shutil
import sys

FILES = ('run.py', 'LICENSE', 'lib/nerf_utils.py', 'lib/ops.py', 'lib/pose_utils.py',
         'models/generator.py', 'models/stylegan.py')

DEST = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_ref')
SRC = os.environ.get('NFI_REFERENCE_SRC', '/root/reference')


def stage(src=SRC, dest=DEST, quiet=False):
    """Copies FILES from ``src`` to ``dest``; returns the manifest (path -> sha256)."""
    if not os.path.isfile(os.path.join(src, 'run.py')):
        raise FileNotFoundError('no reference checkout at %s' % src)
    manifest = {}
    for rel in FILES:
        s, d = os.path.join(src, rel), os.path.join(dest, rel)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        shutil.copyfile(s, d)
        with open(d, 'rb') as f:
            manifest[rel] = hashlib.sha256(f.read()).hexdigest()
    with open(os.path.join(dest, 'MANIFEST.json'), 'w') as f:
        json.dump({'source': src, 'files': manifest}, f, indent=1, sort_keys=True)
    if not quiet:
        print('staged %d reference files into %s' % (len(manifest), dest))
    return manifest


if __name__ == '__main__':
    stage(*(sys.argv[1:2] or [SRC]))
