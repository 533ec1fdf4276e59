"""Install the reference's bootstrap encoder for the comparisons -- TEST / BASELINE INFRASTRUCTURE.

Copies the files the reference's ``BootstrapEncoder`` imports (models/encoder.py, the SegFormer it
builds, and lib/utils.py, which that imports) UNMODIFIED from a checkout of
google-research/nerf-from-image into the same git-ignored ``oracle/_ref/`` that
``oracle/stage_reference.py`` fills, beside the files it stages.  They import torch and numpy only,
and ``pretrained=False`` needs no SegFormer checkpoint.

Used by: ``__graft_entry__.build()`` (after ``stage_reference.stage``, where a reference checkout
exists), then by tests/encoder_standin.py's ``reference_encoder`` -> tests/test_encoder_*.py and
tools/time_encoder_step.py.  Without it those comparisons fall back to the committed golden vectors
or to the stand-in module.
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

FILES = ('models/encoder.py', 'models/segformer.py', 'lib/utils.py')


def stage(src=stage_reference.SRC, dest=stage_reference.DEST, quiet=False):
    """Copies FILES from ``src`` to ``dest``; returns the manifest (path -> sha256)."""
    if not all(os.path.isfile(os.path.join(src, rel)) for rel in FILES):
        raise FileNotFoundError('no reference encoder sources at %s' % src)
    manifest = {}
    for rel in FILES:
        s, d = os.path.join(src, rel), os.path.join(dest, rel)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        shutil.copyfile(s, d)
        with open(d, 'rb') as f:
            manifest[rel] = hashlib.sha256(f.read()).hexdigest()
    with open(os.path.join(dest, 'MANIFEST.encoder.json'), 'w') as f:
        json.dump({'source': src, 'files': manifest}, f, indent=1, sort_keys=True)
    if not quiet:
        print('staged %d reference encoder files into %s' % (len(manifest), dest))
    return manifest


def available(root):
    """Whether ``root`` (a staged or checked-out reference) has the encoder's files."""
    return all(os.path.isfile(os.path.join(root, rel)) for rel in FILES)


if __name__ == '__main__':
    stage(*(sys.argv[1:2] or [stage_reference.SRC]))
