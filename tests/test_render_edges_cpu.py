"""The float64 Path R reference of tests/render_ref64.py, checked without a GPU: against the float32 numpy oracle
(oracle/warp_oracle.py) and against the goldens minted from the reference's own code (tests/golden/warp_R*.npz,
warp_cache.npz).  The per-pixel bound and guard band are the ones the GPU tests hold the kernels to; the oracle is
an fp32 evaluation of the same arithmetic with IEEE exp / log1p, so it must sit inside the "exact" bound."""
import numpy as np
import pytest

from oracle import cases, golden, warp_oracle

from . import render_ref64 as ref

F32 = np.float32


def _check_item(r, out, mask, depth=None, guard_max=0.05, same_positions=False):
    """Every texel outside the guard band within the bound; masks equal outside it.  Returns (worst ratio, guard).
    same_positions: the positions are the checked implementation's own, so only the tiny-weight texels are guarded
    (no knife edge can flip an index)."""
    g = r["tiny"] if same_positions else r["guard"]
    assert g.mean() <= guard_max, g.mean()
    assert np.array_equal((mask > 0)[~g], (r["mask"] > 0)[~g])
    worst = ref.excess(out, r["out"], r["bound"], g)
    if depth is not None:
        worst = max(worst, ref.excess(depth, r["depth"], r["dbound"], g | (r["mask"] == 0)))
    return worst, float(g.mean())


@pytest.mark.parametrize("h,w", [(1, 1), (2, 3), (5, 13), (13, 8), (24, 32)])
@pytest.mark.parametrize("is_image", [True, False])
def test_splat_reference_matches_oracle(h, w, is_image):
    """bilinear_splatting: random sub-pixel flow reaching into the ring and past W + 1 / H + 1, a dolly-out
    cluster, fractional mask, depths over two decades."""
    rng = np.random.RandomState(h * 100 + w + int(is_image))
    C = 3
    frame = rng.uniform(-1, 1, (1, C, h, w)).astype(F32)
    mask = rng.uniform(0, 1, (1, 1, h, w)).astype(F32)
    depth = np.exp(rng.uniform(-1, 3, (1, 1, h, w))).astype(F32)
    flow = rng.uniform(-2.5, 2.5, (1, 2, h, w)).astype(F32)
    flow[:, :, : h // 2, : w // 2] = (np.array([w / 2 - 0.3, h / 2 + 0.2], F32).reshape(1, 2, 1, 1)
                                      - warp_oracle.create_grid(1, h, w)[:, :, : h // 2, : w // 2])
    o, m = warp_oracle.bilinear_splatting(frame, mask, depth, flow, is_image=is_image)
    lz = np.log1p(depth.astype(np.float64)).max()
    r = ref.splat(frame[0], mask[0, 0], depth[0, 0].astype(np.float64), flow[0], lz, path="exact", is_image=is_image)
    worst, _ = _check_item(r, o[0], m[0, 0], same_positions=True)
    assert worst <= 1.0, worst


@pytest.mark.parametrize("name", ["R1", "R2", "R3", "R4", "R5", "R6"])
def test_forward_warp_reference_matches_golden(name, golden_dir):
    """The reference's own forward_warp (the golden) on its own flow and world points."""
    g = golden.load(golden_dir, f"warp_{name}")
    c = cases.warp_case(name)
    b = c["image"].shape[0]
    masks = None if c["mask"] is None else c["mask"][:, 0]
    res = ref.forward_warp(c["image"], masks, g["points"], c["w2c_tgt"], c["K"], g["flow"], "exact")
    for i in range(b):
        worst, guard = _check_item(res[i], g["warped"][i], g["mask"][i, 0], g["depth"][i], same_positions=True)
        assert worst <= 1.0, (i, worst)


def test_render_cache_reference_matches_golden(golden_dir):
    """Cache3D render (N = 2, F = 3, chunks of two items sharing a max) on positions from the oracle's fp32 flow."""
    g = golden.load(golden_dir, "warp_cache")
    c = cases.warp_case("R3")
    F, N = 3, 2
    w2cs = cases.pan_trajectory(F, 0.1)
    K = c["K"][0]
    pts = g["points"][0, 0]                       # (N, H, W, 3)
    img = c["image"]                              # (N, 3, H, W)
    msk = g["cache_mask"][0, 0, :, 0]
    items = [(f, n) for f in range(F) for n in range(N)]
    P = np.stack([pts[n] for f, n in items])
    I = np.stack([img[n] for f, n in items])
    M = np.stack([msk[n] for f, n in items])
    Wc = np.stack([w2cs[f] for f, n in items]).astype(F32)
    Kc = np.stack([K for _ in items])
    _, _, _, flows = warp_oracle.forward_warp(I, M[:, None], P, Wc, Kc)
    res = ref.forward_warp(I, M, P, Wc, Kc, flows, "exact", group=2, foreign_flow=True)
    for j, (f, n) in enumerate(items):
        worst, _ = _check_item(res[j], g["pixels"][0, f, n], g["masks"][0, f, n, 0])
        assert worst <= 1.0, (f, n, worst)


def test_flow_bound_holds_for_the_oracle_projection():
    c = cases.warp_case("R2")
    pts = warp_oracle.unproject_points(c["depth"], c["w2c_src"], c["K"])
    _, _, _, flow = warp_oracle.forward_warp(c["image"], None, pts, c["w2c_tgt"], c["K"])
    for i in range(pts.shape[0]):
        q, qe = ref.project64(pts[i], c["w2c_tgt"][i], c["K"][i])
        f64, ferr = ref.flow64(q, qe, *pts.shape[1:3])
        ok = q[..., 2] > 1e-3
        assert (np.abs(flow[i] - f64) <= ferr)[:, ok].all()


CONTROLS = {"crop_shift": dict(crop_shift=1), "per_item_max": dict(per_item_max=True),
            "ignore_mask": dict(ignore_mask=True), "swap_ne_sw": dict(swap_ne_sw=True), "no_soft_z": dict(soft_z=False)}


@pytest.mark.parametrize("control", list(CONTROLS))
def test_negative_controls_miss_the_oracle(control):
    """Each deliberate error in the reference misses the bar against the oracle on the same data."""
    c = cases.warp_case("R3")
    h, w = 24, 32
    pts = warp_oracle.unproject_points(c["depth"][:, :, :h, :w], c["w2c_src"], c["K"])
    pts = np.concatenate([pts[:1], pts[:1] * F32(0.5)])     # two items of different depth range: one shared max
    img = np.ascontiguousarray(c["image"][:, :, :h, :w])
    rng = np.random.RandomState(1)
    mask = (rng.uniform(0, 1, (2, 1, h, w)) > 0.3).astype(F32) * rng.uniform(0.2, 1, (2, 1, h, w)).astype(F32)
    w2c, K = c["w2c_tgt"], c["K"]
    o, m, _, flow = warp_oracle.forward_warp(img, mask, pts, w2c, K)
    good = ref.forward_warp(img, mask[:, 0], pts, w2c, K, flow, "exact")
    bad = ref.forward_warp(img, mask[:, 0], pts, w2c, K, flow, "exact", **CONTROLS[control])
    assert max(_check_item(good[i], o[i], m[i, 0])[0] for i in range(2)) <= 1.0
    worst = 0.0
    for i in range(2):
        g = good[i]["guard"]
        worst = max(worst, ref.excess(o[i], bad[i]["out"], good[i]["bound"], g),
                    float(((m[i, 0] > 0) != (bad[i]["mask"] > 0))[~g].any()) * 1e9)
    assert worst > 10.0, worst


@pytest.mark.parametrize("window", [1, 3, 5, 7])
@pytest.mark.parametrize("h,w", [(2, 3), (6, 5), (24, 32)])
def test_reliable_mask_reference_matches_oracle(window, h, w):
    rng = np.random.RandomState(window + h)
    d = (2 + rng.uniform(0, 0.2, (h, w))).astype(F32)
    d[rng.uniform(0, 1, (h, w)) < 0.1] = 0
    o = warp_oracle.reliable_depth_mask_range_batch(d[None, None], window, 0.05)[0, 0]
    m, g = ref.reliable64(d, window, 0.05)
    assert np.array_equal(o[~g], m[~g]) and g.mean() < 0.05


@pytest.mark.parametrize("is_depth", [True, False])
def test_unproject_reference_matches_oracle(is_depth):
    c = cases.warp_case("R4")
    d = c["depth"][:1, :, :20, :24].copy()
    d[0, 0, 3, :5] = 0
    d[0, 0, 4, :5] = -1
    o = warp_oracle.unproject_points(d, c["w2c_src"][:1], c["K"][:1], is_depth=is_depth)[0]
    p, bnd, valid = ref.unproject64(d[0, 0], c["w2c_src"][0], c["K"][0], is_depth)
    assert (o[~valid] == 0).all()
    # the oracle inverts in fp32 (torch.linalg.inv) and multiplies in another order: a few more ulp than the kernel
    assert (np.abs(o - p) <= 4 * bnd + 1e-30).all()
