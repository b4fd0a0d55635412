"""CPU model of the attention kernel's online softmax with its lazy rescale (gen3c_b200/csrc/attn_wgmma.cu,
softmax_tile): exact row max per 128-key tile; the reference m of the rows of one warp (16 consecutive query rows)
moves — with O and the row sums rescaled by 2^(m_old - m_new) — only when some row of the warp exceeds its m by more
than 8 (log2 units); the first tile always sets m.  Run step by step in float32 with P rounded to bf16 for the P.V
product, the model must match an fp64 softmax on the cases the GPU tests build (tests/test_attn_lazy_rescale_gpu.py),
and the two rules the kernel must not use — comparing with the previous tile's max, or letting one row decide for the
warp — must fail on them."""
import numpy as np
import pytest
import torch

TILE, WARP_ROWS, THRESHOLD = 128, 16, 8.0


def bf16(x: np.ndarray) -> np.ndarray:
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).float().numpy()


def kernel_model(S: np.ndarray, V: np.ndarray, rule: str = "warp") -> np.ndarray:
    """S [rows, keys] float32 scores in log2 units (keys a multiple of 128, rows of 16), V [keys, d] -> O / l.
    rule: "warp" (the kernel), "previous_tile" (growth against the last tile's max), "first_row" (row 0 of the warp
    decides)."""
    rows, keys = S.shape
    m = np.full(rows, -np.inf, np.float32)
    prev = np.full(rows, -np.inf, np.float32)
    l = np.zeros(rows, np.float32)
    O = np.zeros((rows, V.shape[1]), np.float32)
    for j in range(keys // TILE):
        s = S[:, j * TILE:(j + 1) * TILE]
        mx = s.max(axis=1)
        with np.errstate(invalid="ignore"):
            grow = mx - (prev if rule == "previous_tile" else m) > THRESHOLD
        grow |= np.isneginf(m)
        grow = grow.reshape(-1, WARP_ROWS)
        move = np.repeat(grow[:, 0] if rule == "first_row" else grow.any(axis=1), WARP_ROWS)
        nm = np.where(move, np.maximum(m, mx), m)
        with np.errstate(invalid="ignore", over="ignore"):
            alpha = np.where(move, np.exp2(m - nm), 1.0).astype(np.float32)
            l *= alpha
            O *= alpha[:, None]
            m, prev = nm, mx
            p = np.exp2(s - m[:, None]).astype(np.float32)
            l = l + p.sum(axis=1, dtype=np.float32)
            O = O + bf16(p) @ V[j * TILE:(j + 1) * TILE]
    with np.errstate(invalid="ignore"):
        return O / l[:, None]


def exact(S, V):
    s = S.astype(np.float64)
    p = np.exp2(s - s.max(axis=1, keepdims=True))
    return (p / p.sum(axis=1, keepdims=True)) @ V.astype(np.float64)


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def case(name, rng):
    rows = 64
    if name == "staircase":   # +4 per tile over 55 tiles
        keys = 55 * TILE
        S = rng.standard_normal((rows, keys)) * 0.1 + 4.0 * (np.arange(keys) // TILE) - 1.0
        S[:, np.arange(55) * TILE + 77] = 4.0 * np.arange(55)
    elif name == "divergent":  # one row of warp 2 jumps by 150 in tile 2
        keys = 5 * TILE
        S = rng.standard_normal((rows, keys)) * 0.1 - 1.0
        S[45, 2 * TILE + 9] = 150.0
    elif name.startswith("edge"):  # 16 keys `rise` above the first tile's max in tile 3
        keys = 8 * TILE
        S = rng.standard_normal((rows, keys)) * 0.1 - 1.0
        S[:, 5] = 0.0
        S[:, 3 * TILE + 40:3 * TILE + 56] = float(name[4:])
    else:  # "wild": logits over +-250
        keys = 16 * TILE
        S = rng.standard_normal((rows, keys)) * 75.0
    return S.astype(np.float32), bf16(rng.standard_normal((keys, 128)))


@pytest.mark.parametrize("name", ["staircase", "divergent", "edge7.9", "edge8.0", "edge8.1", "wild"])
def test_lazy_rescale_matches_exact(name):
    S, V = case(name, np.random.default_rng(7))
    out = kernel_model(S, V)
    assert np.isfinite(out).all()
    assert rel(out, exact(S, V)) < 4e-3


def test_p_stays_below_threshold_between_moves():
    """Between moves P = 2^(s - m) <= 2^8: bf16 holds it exactly at the bound and the fp32 sums have 2^119 to spare."""
    S, V = case("staircase", np.random.default_rng(8))
    m = np.full(S.shape[0], -np.inf, np.float32)
    for j in range(S.shape[1] // TILE):
        mx = S[:, j * TILE:(j + 1) * TILE].max(axis=1)
        move = np.repeat((mx - m > THRESHOLD).reshape(-1, WARP_ROWS).any(axis=1), WARP_ROWS)
        m = np.where(move, np.maximum(m, mx), m)
        assert (S[:, j * TILE:(j + 1) * TILE] - m[:, None]).max() <= THRESHOLD


@pytest.mark.parametrize("rule,name", [("previous_tile", "staircase"), ("first_row", "divergent")])
def test_wrong_rules_fail(rule, name):
    """Negative controls: the staircase never grows by more than 8 from one tile to the next, and in the divergent case
    the jumping row is not row 0 of its warp — both rules leave P = 2^150 or more, which overflows."""
    S, V = case(name, np.random.default_rng(7))
    with np.errstate(over="ignore", invalid="ignore"):
        out = kernel_model(S, V, rule)
        assert not (np.isfinite(out).all() and rel(out, exact(S, V)) < 4e-3)
