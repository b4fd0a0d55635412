"""CPU model of the sum-guarded online softmax, the cheaper alternative to an exact row max per KV tile: exact row max for
the first 128-key tile only, stale reference afterwards, reference shifted by a tile's row-sum exponent when it exceeds
2^40, sticky overflow flag -> exact second pass.  The model runs step by step in float32 (P rounded to bf16 for the P.V
product, as a bf16 MMA operand is) and must agree with an fp64 softmax on benign, drifting and adversarial score
distributions — the same cases the GPU tests run through the C ABI (tests/test_dit_ops_gpu.py).  The attention kernel
(gen3c_b200/csrc/attn_wgmma.cu) uses the exact per-tile row max, i.e. the `exact=True` sweep of this model; the guarded
sweep is kept validated here as the candidate for removing the per-tile max reduction."""
import numpy as np
import pytest
import torch

TILE = 128
BIG = np.float32(2.0 ** 40)
SAFE = np.float32(1e27)


def bf16(x: np.ndarray) -> np.ndarray:
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).float().numpy()


def kernel_model(S: np.ndarray, V: np.ndarray, unit_scale: bool):
    """S [rows, keys] scores in log2 units (float32), V [keys, d].  Returns (O / l, took_second_pass)."""
    rows, keys = S.shape
    nt = keys // TILE

    def sweep(exact: bool):
        ref = np.zeros(rows, np.float32)
        l = np.zeros(rows, np.float32)
        O = np.zeros((rows, V.shape[1]), np.float32)
        pend = np.zeros(rows, np.float32)
        ovf = False
        for j in range(nt):
            s = S[:, j * TILE:(j + 1) * TILE]
            if exact or j == 0:
                mx = s.max(axis=1)
                if j == 0:
                    plain = (not exact) and unit_scale and bool(np.all(np.abs(mx) <= 40.0))
                    ref = np.zeros(rows, np.float32) if plain else mx.copy()
                elif np.any(mx - ref > 8.0):  # lazy rescale, warp-wide decision modelled as global
                    nref = np.maximum(ref, mx)
                    alpha = np.exp2(ref - nref).astype(np.float32)
                    l *= alpha
                    O *= alpha[:, None]
                    ref = nref
            elif np.any(pend != 0):
                alpha = np.exp2(-pend).astype(np.float32)
                l *= alpha
                O *= alpha[:, None]
                ref = ref + pend
                pend = np.zeros(rows, np.float32)
            with np.errstate(over="ignore", invalid="ignore"):
                p = np.exp2((s - ref[:, None]).astype(np.float32)).astype(np.float32)
                tsum = p.sum(axis=1, dtype=np.float32)
                l = l + tsum
                O = O + bf16(p) @ V[j * TILE:(j + 1) * TILE]
            if not exact:
                ovf = ovf or bool(np.any(~(l < SAFE)))
                e = ((tsum.view(np.int32) >> 23) & 0xFF) - 127
                pend = np.where(tsum > BIG, np.minimum(e, 100), 0).astype(np.float32)
        return O, l, ovf

    O, l, ovf = sweep(exact=False)
    second = ovf or bool(np.any(~(l < SAFE)))
    if second:
        O, l, _ = sweep(exact=True)
    return O / l[:, None], second


def exact(S, V):
    s = S.astype(np.float64)
    p = np.exp2(s - s.max(axis=1, keepdims=True))
    return (p / p.sum(axis=1, keepdims=True)) @ V.astype(np.float64)


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.mark.parametrize("case,second", [("benign", False), ("drift", False), ("jump65", False), ("jump155", True),
                                         ("wild", True)])
def test_guarded_softmax_matches_exact(case, second):
    rng = np.random.default_rng(5)
    rows, keys, d = 64, 2048, 128
    V = bf16(rng.standard_normal((keys, d)))
    S = (rng.standard_normal((rows, keys)) * 1.5).astype(np.float32)
    if case == "drift":      # maxima grow by ~2^60 over the sweep: absorbed by exponent shifts, never a second pass
        S += np.linspace(0, 60, keys, dtype=np.float32)[None, :]
    elif case == "jump65":   # one block of keys 2^65 above everything before it (GPU test jump=4.0)
        S[:, 300:340] += 65.0
    elif case == "jump155":  # 2^155: overflows inside that tile (GPU test jump=9.5)
        S[:, 300:340] += 155.0
    elif case == "wild":     # logits spread over +-250 (GPU test gain=6.0): transient l ~ 1e38 behind a later shift
        S = (rng.standard_normal((rows, keys)) * 75.0).astype(np.float32)
    out, took_second = kernel_model(S, V, unit_scale=True)
    assert np.isfinite(out).all()
    assert took_second == second
    assert rel(out, exact(S, V)) < 4e-3
