"""Record the reference's compute_pose_pnp outputs on the PnP fixtures (tests/pnp_cases.py) as
tests/golden/reference/pnp_<case>.npz, for machines without cv2 -- TEST INFRASTRUCTURE.

Needs cv2 and the staged reference (oracle/stage_pnp_reference.py).  Run from the repository root:
``python -m oracle.record_pnp_reference``."""
import os

import numpy as np

from oracle import stage_pnp_reference
from tests import pnp_cases

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden',
                   'reference')


def main():
    import cv2
    ref = stage_pnp_reference.reference_compute_pose_pnp()
    if ref is None:
        raise SystemExit('the staged reference or cv2 is missing')
    for name, (co, m, f, refine) in pnp_cases.cases().items():
        w, fo, e = ref(co, m, f, refine=refine)
        np.savez(os.path.join(OUT, 'pnp_%s.npz' % name), world2cam=w, focal=np.asarray(fo, np.float64),
                 error=np.asarray(e, np.float64), cv2_version=cv2.__version__)
        print(name, 'recorded')


if __name__ == '__main__':
    main()
