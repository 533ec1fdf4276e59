"""Install the reference's discriminator for the comparisons -- TEST / BASELINE INFRASTRUCTURE.

Copies models/discriminator.py (the ``Discriminator`` that run.py builds) UNMODIFIED from a checkout
of google-research/nerf-from-image into the same git-ignored ``oracle/_ref/`` that
``oracle/stage_reference.py`` fills.  Its imports, models/stylegan.py and lib/pose_utils.py, are
among the files that script stages.

Used by: ``__graft_entry__.build()`` (after ``stage_reference.stage``, where a reference checkout
exists), then by tests/test_disc_*.py and tools/time_discriminator.py.  Without it those
comparisons fall back to the committed golden vectors (tests/golden/reference/) or skip.
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

FILES = ('models/discriminator.py',)


def stage(src=stage_reference.SRC, dest=stage_reference.DEST, quiet=False):
    """Copies FILES from ``src`` to ``dest``; returns the manifest (path -> sha256)."""
    if not available(src):
        raise FileNotFoundError('no reference discriminator source at %s' % src)
    manifest = {}
    for rel in FILES:
        s, d = os.path.join(src, rel), os.path.join(dest, rel)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        shutil.copyfile(s, d)
        with open(d, 'rb') as f:
            manifest[rel] = hashlib.sha256(f.read()).hexdigest()
    with open(os.path.join(dest, 'MANIFEST.disc.json'), 'w') as f:
        json.dump({'source': src, 'files': manifest}, f, indent=1, sort_keys=True)
    if not quiet:
        print('staged %d reference discriminator file into %s' % (len(manifest), dest))
    return manifest


def available(root):
    """Whether ``root`` (a staged or checked-out reference) has the discriminator's file."""
    return all(os.path.isfile(os.path.join(root, rel)) for rel in FILES)


if __name__ == '__main__':
    stage(*(sys.argv[1:2] or [stage_reference.SRC]))
