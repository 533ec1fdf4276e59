"""Times the inversion's pose initialisation: the fused estimate_poses_batch (nfi_pnp.cu) at B = 16
and 64, 128^2, 11 focal guesses, with CUDA events after warm-up; and the reference's host path
(OpenCV) on the same machine's cores where cv2 and the staged reference exist.  Prints the card and
its power limit from the same run; with a path argument also writes the JSON there."""
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from nerf_from_image_b200 import pnp  # noqa: E402
from oracle import stage_pnp_reference  # noqa: E402
from tests import pnp_cases as C  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def time_fused(co, m, reps=20):
    cot, mt = torch.from_numpy(co).cuda(), torch.from_numpy(m.astype(np.float32)).cuda()
    for _ in range(3):
        pnp.estimate_poses_batch(cot, mt, C.FOCAL_GUESSES)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        pnp.estimate_poses_batch(cot, mt, C.FOCAL_GUESSES)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return ms


def time_reference(co, m, reps=3):
    ref = stage_pnp_reference.reference_compute_pose_pnp()
    if ref is None:
        return None
    out = []
    for _ in range(reps):
        t = time.perf_counter()
        ref(co, m, C.FOCAL_GUESSES)
        out.append((time.perf_counter() - t) * 1e3)
    return out



def local_memory_mib():
    """Device memory the first solve takes beyond PyTorch's allocations: the driver's local-memory
    reservation for solve_kernel's per-thread stack frame."""
    co, m, _ = C.ellipsoid_views(0, 1, res=32, focal=2.0)
    cot, mt = torch.from_numpy(co).cuda(), torch.from_numpy(m).cuda()
    torch.cuda.synchronize()
    free0, res0 = torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved()
    pnp.compute_pose_pnp(cot, mt, [2.0])
    torch.cuda.synchronize()
    free1, res1 = torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved()
    return ((free0 - free1) - (res1 - res0)) / 2 ** 20


def main():
    torch.zeros(1, device='cuda')
    res = {'card': card(), 'cpu_count': os.cpu_count(), 'local_memory_mib': local_memory_mib()}
    for b in (16, 64):
        co, m, _ = C.ellipsoid_views(b, b, res=128, focal=2.0)
        ms = time_fused(co, m)
        res['fused_B%d_ms' % b] = {'median': statistics.median(ms), 'min': min(ms), 'max': max(ms)}
        r = time_reference(co, m)
        res['reference_B%d_ms' % b] = ({'median': statistics.median(r), 'min': min(r), 'max': max(r)}
                                       if r else 'not measured')
        res['foreground_pixels_mean_B%d' % b] = float(m.reshape(b, -1).sum(1).mean())
    print(json.dumps(res, indent=1))
    if len(sys.argv) > 1:
        with open(sys.argv[1], 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
