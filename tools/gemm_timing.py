"""Time every Linear of a DiT block with the epilogue the engine gives it, at M = 56 320 tokens (the benchmark's
latent), next to the plain f32 / bf16 epilogues and cuBLAS (torch.mm, bf16) on the same seeded operands:

  * to_q / to_k: per-head RMSNorm + RoPE with a cos|sin table;  CA to_q: the norm alone
  * V^T: the same kernel with the operands swapped ([D, M] output)
  * FA / CA to_out (K = D) and layer2 (K = F): x += gate * acc on an fp32 residual x
  * layer1: GELU

Each row runs back to back for at least --seconds of device time.  Prints a table and one JSON object (written to
DIR/gemm_timing.json with --out), with the card name, power limit and SM clock read in the same run.

    python tools/gemm_timing.py [--out DIR] [--dump DIR [--dump-rows R]]
    python tools/gemm_timing.py --compare DIR_A DIR_B

--dump writes the first R rows of each launch's output (one launch on fresh operands) as DIR/<row>.pt; --compare
reports, for two such dumps, which outputs are bit-identical and, for the gated residual, the largest difference in
units of one rounding of the product gate * acc plus one of the sum.  Needs an H100 for everything but --compare."""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

M_TOKENS, D, F = 16 * 44 * 80, 4096, 16384
# launches of each gated residual per denoise step: 28 blocks x 2 forwards (conditional, unconditional)
GATED_PER_STEP = {"to_out": 2 * 56, "layer2": 56}


def time_row(torch, fn, seconds):
    """ms per launch over back-to-back launches lasting at least `seconds` (CUDA events)."""
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    iters = max(10, math.ceil(seconds * 1e3 / max(s.elapsed_time(e), 1e-3)))
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters, iters


def run(args):
    import torch

    from fp8_timing import card
    from gen3c_b200 import ops

    assert torch.cuda.is_available(), "needs a CUDA device"
    torch.cuda.set_device(0)
    result = {"card_before": card(), "M": M_TOKENS, "rows": {}}
    g = torch.Generator(device="cuda").manual_seed(0)
    dev = "cuda"

    def randn(*shape, scale=1.0):
        return scale * torch.randn(*shape, device=dev, generator=g)

    gamma = (1.0 + randn(128, scale=0.1)).contiguous()
    ang = torch.rand(M_TOKENS, 64, device=dev, generator=g) * (2 * math.pi)
    cs = torch.cat([ang.cos(), ang.sin()], 1).contiguous()
    gate = randn(D, scale=0.1).contiguous()
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)

    def dump(name, t):
        if args.dump:
            torch.save(t[: args.dump_rows].cpu().clone(), os.path.join(args.dump, name + ".pt"))

    # operand set -> (M, N, K, [(row name, epilogue)])
    sets = {
        "qkvo": (M_TOKENS, D, D, ["norm_rope", "norm", "gated", "f32", "bf16", "cublas"]),
        "vt": (D, M_TOKENS, D, ["bf16", "f32", "cublas"]),
        "layer1": (M_TOKENS, F, D, ["gelu", "f32", "bf16", "cublas"]),
        "layer2": (M_TOKENS, D, F, ["gated", "f32", "bf16", "cublas"]),
    }
    for sname, (m, n, k, epis) in sets.items():
        a = randn(m, k).to(torch.bfloat16)
        b = randn(n, k, scale=k ** -0.5).to(torch.bfloat16)
        flop = 2.0 * m * n * k
        x0 = randn(m, n) if "gated" in epis else None
        for epi in epis:
            if epi in ("bf16", "gelu", "norm_rope", "norm", "cublas"):
                out = torch.empty(m, n, device=dev, dtype=torch.bfloat16)
            else:
                out = torch.empty(m, n, device=dev, dtype=torch.float32)
            if epi == "norm_rope":
                fn = lambda: ops.gemm_norm_rope(a, b, gamma, cs)  # noqa: E731
            elif epi == "norm":
                fn = lambda: ops.gemm_norm_rope(a, b, gamma, None)  # noqa: E731
            elif epi == "gated":
                fn = lambda: ops.gemm(a, b, ops.EPI_GATED_RESIDUAL_F32, out=out, gate=gate)  # noqa: E731
            elif epi == "cublas":
                fn = lambda: torch.mm(a, b.t(), out=out)  # noqa: E731
            else:
                code = {"bf16": ops.EPI_BF16, "gelu": ops.EPI_GELU_BF16, "f32": ops.EPI_F32}[epi]
                fn = lambda code=code: ops.gemm(a, b, code, out=out)  # noqa: E731
            if args.dump and epi != "cublas":
                if epi == "gated":
                    out.copy_(x0)
                    fn()
                    dump(f"{sname}.x0", x0)
                    dump(f"{sname}.gate", gate[None, :])
                    dump(f"{sname}.{epi}", out)
                else:
                    dump(f"{sname}.{epi}", fn())
            if epi == "gated":
                out.copy_(x0)
            ms, iters = time_row(torch, fn, args.seconds)
            row = {"M": m, "N": n, "K": k, "ms": ms, "tflops": flop / (ms * 1e-3) / 1e12, "launches": iters}
            result["rows"][f"{sname}.{epi}"] = row
            print(f"{sname:7s} {epi:10s} M={m:6d} N={n:6d} K={k:6d}  {ms:8.3f} ms  {row['tflops']:6.1f} TFLOP/s",
                  flush=True)
            del out
        del a, b, x0
        torch.cuda.empty_cache()
    rows = result["rows"]
    gap = {"to_out": rows["qkvo.gated"]["ms"] - rows["qkvo.f32"]["ms"],
           "layer2": rows["layer2.gated"]["ms"] - rows["layer2.f32"]["ms"]}
    result["gated_minus_f32_ms"] = gap
    result["gated_minus_f32_ms_per_step"] = sum(GATED_PER_STEP[k] * v for k, v in gap.items())
    result["card_after"] = card()
    txt = json.dumps(result, indent=1)
    print(txt)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "gemm_timing.json"), "w") as f:
            f.write(txt)


def compare(dir_a, dir_b):
    import torch

    res = {}
    for fn in sorted(os.listdir(dir_a)):
        name = fn[:-3]
        if not fn.endswith(".pt") or name.endswith((".x0", ".gate")):
            continue
        a, b = torch.load(os.path.join(dir_a, fn)), torch.load(os.path.join(dir_b, fn))
        r = {"bit_identical": bool(torch.equal(a.view(torch.int16 if a.dtype == torch.bfloat16 else torch.int32),
                                               b.view(torch.int16 if b.dtype == torch.bfloat16 else torch.int32))),
             "differing": int((a != b).sum())}
        if name.endswith(".gated"):
            s = name.split(".")[0]
            acc = torch.load(os.path.join(dir_a, f"{s}.f32.pt")).double()
            g = torch.load(os.path.join(dir_a, f"{s}.gate.pt")).double()
            prod = (g * acc).abs()
            d = (a.double() - b.double()).abs()
            # one rounding of gate * acc (2^-24 |p|), and the sums rounded apart by up to one ulp (2^-23 |x_new|)
            bound = 2.0 ** -24 * prod + 2.0 ** -23 * torch.maximum(a.double().abs(), b.double().abs())
            r["max_abs_diff"] = float(d.max())
            r["max_diff_over_one_rounding"] = float((d / bound.clamp_min(1e-38)).max())
        res[name] = r
        print(name, r, flush=True)
    print(json.dumps(res, indent=1))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.2, help="least device time per row")
    ap.add_argument("--out", default=None)
    ap.add_argument("--dump", default=None, metavar="DIR")
    ap.add_argument("--dump-rows", type=int, default=1 << 30)
    ap.add_argument("--compare", nargs=2, default=None, metavar=("DIR_A", "DIR_B"))
    args = ap.parse_args()
    if args.compare:
        compare(*args.compare)
    else:
        run(args)


if __name__ == "__main__":
    main()
