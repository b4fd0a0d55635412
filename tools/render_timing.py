"""Cost of the ordered (deterministic) Path R splat against the default atomic splat.

    python tools/render_timing.py [--rounds 5] [--renders 5]

Workloads: the benchmark's Path R render (one cached 704 x 1280 frame rendered at 121 poses of a pan) and the same
cache at 121 poses of a dolly-out (the camera backs away to 3 m, so the frame contracts onto fewer texels).  Each round
times `--renders` renders per workload in the default mode, then as many under torch.use_deterministic_algorithms(True),
with CUDA events around the renders.  Prints one JSON line: the median ms per 121-frame render of each workload and
mode over the rounds, their min / max, and the GPU name, power limit and SM clock that nvidia-smi reports (queried
only, nothing is set)."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W, FRAMES = 704, 1280, 121


def smi():
    r = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
                        "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    if r.returncode != 0 or not r.stdout.strip():
        return {}
    f = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": f[0], "power_limit_w": f[1], "sm_clock_mhz": f[2], "sm_clock_max_mhz": f[3]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--renders", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch

    from gen3c_b200 import warp
    from gen3c_b200.cache_3d import Cache3D_Buffer
    from oracle import cases  # synthetic inputs only (seeded depth / trajectory)

    assert torch.cuda.is_available(), "render_timing needs a CUDA device"
    dev = torch.device("cuda", 0)
    img = torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(0)).to(dev) * 2 - 1
    K = torch.from_numpy(cases.intrinsics(H, W)[None]).to(dev)
    cache = Cache3D_Buffer(frame_buffer_max=2, noise_aug_strength=0, generator=None, input_image=img,
                           input_depth=torch.from_numpy(cases.smooth_depth(H, W)[None, None]).to(dev),
                           input_w2c=torch.eye(4, device=dev)[None], input_intrinsics=K, device=dev)
    pts, im = cache.input_points[:, :, :, 0], cache.input_image[:, :, :, 0]
    Ks = K[None].expand(1, FRAMES, 3, 3).contiguous()
    dolly = np.stack([cases.look(0.0, 0.0, (0.0, 0.0, 3.0 * i / (FRAMES - 1))) for i in range(FRAMES)])
    workloads = {"pan": torch.from_numpy(cases.pan_trajectory(FRAMES, 0.3))[None].to(dev),
                 "dolly_out": torch.from_numpy(dolly)[None].to(dev)}

    def timed(w2cs, deterministic):
        torch.use_deterministic_algorithms(deterministic)
        try:
            warp.render_cache(pts, im, None, w2cs, Ks)  # selects the mode on the workspace; warm
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(args.renders):
                warp.render_cache(pts, im, None, w2cs, Ks)
            e.record()
            e.synchronize()
            return s.elapsed_time(e) / args.renders
        finally:
            torch.use_deterministic_algorithms(False)

    times = {f"{w}_{m}": [] for w in workloads for m in ("default", "ordered")}
    for _ in range(args.rounds):
        for w, w2cs in workloads.items():
            times[f"{w}_default"].append(timed(w2cs, False))
            times[f"{w}_ordered"].append(timed(w2cs, True))
    out = {"frames_per_render": FRAMES, "frame": f"{H}x{W}", "rounds": args.rounds, "renders_per_round": args.renders}
    for k, v in times.items():
        out[f"{k}_ms_median"] = statistics.median(v)
        out[f"{k}_ms_min"], out[f"{k}_ms_max"] = min(v), max(v)
    out.update(smi())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
