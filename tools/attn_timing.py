"""Sustained timing of the attention kernel at the benchmark's self-attention shape (Lq = Lk = 56 320, 32 heads, head
dim 128, scale = ln 2), long enough for a power-capped card to settle at its sustained clock.

    python tools/attn_timing.py [--seconds 20] [--trace OUT.json] [--v-layout {vt,tokens}] [--lk LK]

--v-layout vt (the default) times g3c_attn_fwd with V transposed, the engine's layout; tokens times g3c_attn_fwd_sbhd
(gen3c_b200.ops.attention_sbhd, the TE-compatible operator) with V token-major like K.  --lk sets the key count
(default 56 320; 512 is the cross-attention shape).

The library is the one gen3c_b200 loads (GEN3C_B200_LIB selects another build), so two builds are compared by running
this once per build, alternately.  Prints one JSON line: ms per launch, TFLOP/s, the share of the dense-bf16 peak at the
median SM clock that nvidia-smi reported during the timed window (132 SMs x 4096 FLOP/clk), power draw and limit, GPU name.
nvidia-smi is only queried (--query-gpu), nothing is set.  --trace writes the clock64 stamps of CTA (0, 0) of one extra
launch (see g3c_attn_set_trace in include/gen3c_b200.h)."""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

L, HEADS = 56320, 32


def smi_sampler(samples, stop):
    q = "clocks.sm,power.draw,power.limit,name"
    while not stop.is_set():
        r = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
                            f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True)
        if r.returncode == 0 and r.stdout.strip():
            f = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
            samples.append((float(f[0]), float(f[1]), float(f[2]), f[3]))
        stop.wait(0.5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--trace", default=None)
    ap.add_argument("--v-layout", choices=["vt", "tokens"], default="vt")
    ap.add_argument("--lk", type=int, default=L)
    args = ap.parse_args()
    if args.trace and args.v_layout != "vt":
        ap.error("--trace records the V^T kernel only")
    Lk = args.lk
    flop = 4.0 * L * Lk * 128 * HEADS  # Q K^T and P V, 2 FLOP per multiply-add

    import torch

    from gen3c_b200 import _lib, ops

    assert torch.cuda.is_available(), "attn_timing needs a CUDA device"
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(5)
    q, k, v = ((torch.randn(n, HEADS * 128, device=dev, generator=g)).to(torch.bfloat16) for n in (L, Lk, Lk))
    scale = math.log(2.0)
    if args.v_layout == "vt":
        vt = v.T.contiguous()

        def launch():
            return ops.attention(q, k, vt, HEADS, scale=scale)
    else:
        q4, k4, v4 = (t.view(-1, 1, HEADS, 128) for t in (q, k, v))

        def launch():
            return ops.attention_sbhd(q4, k4, v4, scale=scale)

    t_end = time.time() + 3.0  # warm-up: module load, then a few seconds toward the sustained clock
    while time.time() < t_end:
        launch()
        torch.cuda.synchronize()
    samples, stop = [], threading.Event()
    th = threading.Thread(target=smi_sampler, args=(samples, stop), daemon=True)
    th.start()
    times = []
    t_end = time.time() + args.seconds
    while time.time() < t_end:
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(4):
            launch()
        e.record()
        e.synchronize()
        times.append(s.elapsed_time(e) / 4)
    stop.set()
    th.join()
    ms = statistics.median(times)
    tflops = flop / (ms * 1e-3) / 1e12
    out = {"lib": os.environ.get("GEN3C_B200_LIB", str(_lib.LIB_PATH)), "shape": f"{L}x{Lk}, {HEADS} heads, d=128",
           "v_layout": args.v_layout,
           "launches": 4 * len(times), "seconds": args.seconds, "ms_per_launch_median": ms,
           "ms_per_launch_min": min(times), "ms_per_launch_max": max(times), "tflops": tflops}
    if samples:
        clk = statistics.median(x[0] for x in samples)
        peak = 132 * 4096 * clk * 1e6 / 1e12
        out.update({"sm_clock_mhz_median": clk, "power_draw_w_median": statistics.median(x[1] for x in samples),
                    "power_limit_w": samples[0][2], "gpu": samples[0][3], "dense_bf16_peak_at_clock_tflops": peak,
                    "frac_of_peak_at_clock": tflops / peak})
    if args.trace:
        lib = _lib.load()
        buf = torch.zeros(3 * 64 * 8, dtype=torch.int64, device=dev)
        _lib.check(lib.g3c_attn_set_trace(buf.data_ptr()), "g3c_attn_set_trace")
        launch()
        torch.cuda.synchronize()
        _lib.check(lib.g3c_attn_set_trace(None), "g3c_attn_set_trace")
        tr = buf.view(3, 64, 8).cpu()
        t0 = int(tr[1:, :, :5][tr[1:, :, :5] > 0].min())
        rel = {f"consumer{c}": [[int(x) - t0 if x > 0 else None for x in tr[1 + c, j, :5].tolist()] for j in range(64)]
               for c in range(2)}
        with open(args.trace, "w") as f:
            json.dump({"slots": ["turn acquired", "S issued", "S complete", "softmax done", "P.V complete"],
                       "clock64_minus_first": rel}, f)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
