"""Path R per pixel against the float64 reference of tests/render_ref64.py, at the shapes and inputs where the render
branches: every splat kernel, the 1-px ring and its clamps, one-pixel frames, short last passes, the k_project_max
fallback beyond 512 target cameras, occlusion passes after the first, ragged alignment tiles, and the error paths.

Every non-guarded texel of out / mask / depth is held to the derived bound (render_ref64's docstring); each test
prints the worst error as a fraction of the bound and the guard-band fraction (pytest -s shows them).  Branches, by
test id:
  path=points4      k_splat_points4   (W % 4 == 0, 16-byte aligned inputs)
  path=points1_w    k_splat_points    (W % 4 != 0)
  path=points1_align k_splat_points   (W % 4 == 0, inputs a contiguous view at a 4-byte storage offset)
  path=ordered      the ordered splat (k_det_keys .. k_det_accum) under torch.use_deterministic_algorithms
  F=512 / F=513     k_project_max_bcast / its per-item k_project_max fallback (F > PM_MAX_CAM)
  mpp=...           max_items_per_pass: 3 and 4 leave a short last pass
  test_occlusion_passes_after_the_first: foreground_items with > 64 items (item0 of the second pass)
  test_align_*      k_align_step on frames that are not whole 32 x 8 tiles"""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from oracle import cases, warp_oracle

from . import render_ref64 as ref

pytestmark = pytest.mark.gpu

F32 = np.float32
PATHS = ["points4", "points1_w", "points1_align", "ordered"]
# the float64 bound's path: the ordered splat and k_splat_points evaluate the exact expf / log1pf
BOUND_PATH = {"points4": "approx", "points1_w": "exact", "points1_align": "exact", "ordered": "exact"}


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def cu_misaligned(a):
    """A contiguous CUDA copy whose data pointer is 4 bytes past a 16-byte boundary."""
    a = np.ascontiguousarray(a, F32)
    buf = torch.empty(a.size + 1, device="cuda", dtype=torch.float32)
    t = buf[1:].view(a.shape)
    t.copy_(torch.from_numpy(a))
    assert t.is_contiguous() and t.data_ptr() % 16 == 4
    return t


@contextlib.contextmanager
def deterministic(on=True):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def kernels_run(fn):
    """Names of the CUDA kernels fn launches."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}


# ---------------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------------
def target_camera(k):
    """Roll about the optical axis plus a translation: the third row of w2c is (0, 0, 1, t_z), so camera z = p_z + t_z
    exactly in fp32 and a point can sit at z = 0 exactly."""
    a = 0.03 + 0.02 * k
    m = np.eye(4)
    m[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    m[:3, 3] = [0.013 * (k + 1), -0.021, 0.25]
    return m.astype(F32)


def place(K, w2c, u, v, z):
    """The world point that projects to pixel (u, v) at camera depth z."""
    cam = z * (np.linalg.inv(K.astype(np.float64)) @ np.array([u, v, 1.0]))
    m = w2c.astype(np.float64)
    return np.linalg.solve(m[:3, :3], cam - m[:3, 3])


def scene(H, W, b, scale, seed, edges=True):
    """b items of world points (b, H, W, 3) seen by b target cameras.  A smooth depth map times `scale` plus the edge
    geometry: behind the camera, z = 0 exactly and just above, projections into (-1.5, 1.5) and (W - 0.5, W + 2.5) on
    each axis (the clamps into the ring), far off screen, and a dolly-out cluster (many sources on one texel)."""
    rng = np.random.RandomState(seed)
    K = cases.intrinsics(max(H, 2), max(W, 2), f=0.9 * max(H, W) + 3)
    K[0, 2], K[1, 2] = W / 2 - 0.17, H / 2 + 0.11
    src = cases.look(0.02, -0.01, (0.0, 0.0, 0.0))
    pts, w2cs = [], []
    for i in range(b):
        w2c = target_camera(i)
        ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
        d = scale * (2.0 + 0.6 * np.sin(1.3 * xs / max(W, 1) + i) + 0.4 * np.cos(2.1 * ys / max(H, 1)) +
                     0.05 * rng.uniform(-1, 1, (H, W)))
        ray = np.stack([xs, ys, np.ones_like(xs)], -1) @ np.linalg.inv(K.astype(np.float64)).T
        c2w = np.linalg.inv(src.astype(np.float64))
        p = (d[..., None] * ray) @ c2w[:3, :3].T + c2w[:3, 3]
        if edges and H * W >= 12:
            flat = p.reshape(-1, 3)
            sel = rng.permutation(H * W)
            sz = scale * 2.0
            tz = float(w2c[2, 3])
            specials = [place(K, w2c, 0.3 * W, 0.4 * H, -sz),                      # behind the camera
                        np.array([0.1, -0.1, -tz]),                                 # z = 0 exactly
                        np.array([0.0, 0.0, -tz + 1e-6]),                            # just above
                        place(K, w2c, rng.uniform(-1.5, 1.5), 0.5 * H, sz),          # x clamp low
                        place(K, w2c, rng.uniform(W - 0.5, W + 2.5), 0.5 * H, sz),   # x clamp high
                        place(K, w2c, 0.5 * W, rng.uniform(-1.5, 1.5), sz),          # y clamp low
                        place(K, w2c, 0.5 * W, rng.uniform(H - 0.5, H + 2.5), sz),   # y clamp high
                        place(K, w2c, 1e4, -3e3, sz)]                                # far off screen
            for j, q in enumerate(specials):
                flat[sel[j]] = q
            n = max(1, H * W // 8)                                                   # dolly-out cluster
            for j in sel[len(specials):len(specials) + n]:
                flat[j] = place(K, w2c, 0.37 * W + rng.uniform(0, 0.3), 0.61 * H + rng.uniform(0, 0.3),
                                sz * rng.uniform(0.9, 1.1))
        pts.append(p.astype(F32))
        w2cs.append(w2c)
    return np.stack(pts), np.stack(w2cs), np.stack([K] * b).astype(F32)


def run_forward_warp(path, frames, masks, pts, w2cs, Ks, is_image=True, render_depth=True):
    from gen3c_b200 import warp

    put = cu_misaligned if path == "points1_align" else cu
    with deterministic(path == "ordered"):
        w, m, d, f = warp.forward_warp(put(frames), None if masks is None else put(masks[:, None]), None, None,
                                       cu(w2cs), None, cu(Ks), is_image=is_image, render_depth=render_depth,
                                       world_points1=put(pts))
    torch.cuda.synchronize()
    return (w.cpu().numpy(), m.cpu().numpy()[:, 0], None if d is None else d.cpu().numpy(), f.cpu().numpy())


def check_items(res, w, m, d, label):
    """Every non-guarded texel within the bound, masks equal outside the guard band.  Returns (worst, guard)."""
    worst, guard = 0.0, 0.0
    for i, r in enumerate(res):
        g = r["guard"]
        assert np.array_equal(m[i][~g] > 0, r["mask"][~g] > 0), (label, i)
        worst = max(worst, ref.excess(w[i], r["out"], r["bound"], g))
        if d is not None:
            worst = max(worst, ref.excess(d[i], r["depth"], r["dbound"], g | (r["mask"] == 0)))
        guard = max(guard, float(g.mean()))
    print(f"\n[render-edges] {label}: worst/bound {worst:.3g}, guard {guard:.4f}")
    assert worst <= 1.0, (label, worst)
    assert guard <= max(0.05, 5.0 / m[0].size), (label, guard)   # tiny frames: the edge points' few texels
    return worst, guard


FRAMES = {True: [(1, 4), (3, 8), (5, 12), (13, 16), (24, 32), (48, 64)],     # W % 4 == 0
          False: [(1, 1), (2, 3), (5, 13), (8, 13), (13, 5), (37, 50)]}
MASKS = ["none", "fractional", "binary"]


@pytest.mark.parametrize("scale", [1e-2, 1.0, 1e2], ids=lambda s: f"depth{s:g}")
@pytest.mark.parametrize("fi", range(6))
@pytest.mark.parametrize("path", PATHS, ids=lambda p: f"path={p}")
def test_forward_warp_per_pixel(path, fi, scale):
    """forward_warp against float64 on the kernel's own flow; b in {1, 5} (5 > 4 items per pass), C in {1, 2, 3},
    is_image, mask none / fractional / binary, render_depth; the flow against a float64 projection."""
    H, W = FRAMES[path != "points1_w"][fi]
    k = fi + 6 * PATHS.index(path)
    b, C, is_image = (5 if k % 3 == 0 else 1), 1 + k % 3, k % 2 == 0
    mk = MASKS[k % 3]
    rng = np.random.RandomState(k)
    pts, w2cs, Ks = scene(H, W, b, scale, seed=k)
    frames = rng.uniform(-1, 1, (b, C, H, W)).astype(F32)
    masks = None if mk == "none" else rng.uniform(0, 1, (b, H, W)).astype(F32)
    if mk == "binary":
        masks = (masks > 0.3).astype(F32)
    render_depth = k % 4 != 1
    w, m, d, f = run_forward_warp(path, frames, masks, pts, w2cs, Ks, is_image, render_depth)
    res = ref.forward_warp(frames, masks, pts, w2cs, Ks, f, BOUND_PATH[path], is_image=is_image)
    check_items(res, w, m, d, f"forward_warp {path} {H}x{W} b={b} C={C} image={is_image} mask={mk} depth*{scale:g}")
    for i, r in enumerate(res):
        ok = r["z"] > r["zerr"]
        assert (np.abs(f[i] - r["flow"]) <= r["flow_err"])[:, ok].all()


@pytest.mark.parametrize("path", PATHS, ids=lambda p: f"path={p}")
def test_splat_branch_taken(path):
    """The parametrisation reaches the kernel its name says."""
    H, W = (8, 13) if path == "points1_w" else (8, 16)
    pts, w2cs, Ks = scene(H, W, 1, 1.0, seed=1)
    frames = np.zeros((1, 3, H, W), F32)
    names = kernels_run(lambda: run_forward_warp(path, frames, None, pts, w2cs, Ks))
    want = {"points4": "k_splat_points4", "points1_w": "k_splat_points", "points1_align": "k_splat_points",
            "ordered": "k_det_accum"}[path]
    hits = {n for n in names if want in n and not (want == "k_splat_points" and "k_splat_points4" in n)}
    assert hits, (path, names)


def test_approximate_log_depth_against_the_exact_path():
    """The same scene through k_splat_points4 and through k_splat_points (misaligned copy) at three depth scales:
    identical masks, outputs within the sum of both paths' bounds.  Prints the relative weight error the
    approximations cost at each scale (DESIGN.md §3.4)."""
    H, W = 24, 32
    for scale in (1e-2, 1.0, 1e2):
        pts, w2cs, Ks = scene(H, W, 1, scale, seed=5)
        frames = np.random.RandomState(5).uniform(-1, 1, (1, 3, H, W)).astype(F32)
        a = run_forward_warp("points4", frames, None, pts, w2cs, Ks)
        b = run_forward_warp("points1_align", frames, None, pts, w2cs, Ks)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[3], b[3])
        ra = ref.forward_warp(frames, None, pts, w2cs, Ks, a[3], "approx")[0]
        rb = ref.forward_warp(frames, None, pts, w2cs, Ks, a[3], "exact")[0]
        g = ra["guard"]
        ex = ref.excess(a[0][0], b[0][0], ra["bound"] + rb["bound"], g)
        ea = ref.excess(a[0][0], ra["out"], ra["bound"], g)
        eb = ref.excess(b[0][0], rb["out"], rb["bound"], g)
        print(f"\n[render-edges] depth*{scale:g}: approx d_w max {ra['dw'][ra['mask'] > 0].max():.3g}, exact "
              f"{rb['dw'][rb['mask'] > 0].max():.3g}; worst/bound approx {ea:.3g}, exact {eb:.3g}, between {ex:.3g}")
        assert ex <= 1.0 and ea <= 1.0 and eb <= 1.0


def test_nan_and_inf_points():
    """A NaN world point is dropped: its projected depth fails q_z > 0 and log_depth's fmaxf(NaN, 0) = 0 keeps it
    out of the log-depth max, so the render equals the render with that point moved behind the camera (the oracle's
    np.maximum, like torch, would turn every weight of the chunk into NaN instead).  A point at +Inf projects to NaN
    (0 * Inf in the matrix products) and is dropped the same way."""
    H, W = 8, 16
    pts, w2cs, Ks = scene(H, W, 2, 1.0, seed=3, edges=False)
    frames = np.random.RandomState(3).uniform(-1, 1, (2, 3, H, W)).astype(F32)
    behind = pts.copy()
    behind[0, 3, 5] = place(Ks[0], w2cs[0], 4.0, 4.0, -1.0)
    for bad in (np.nan, np.inf):
        odd = pts.copy()
        odd[0, 3, 5] = [0.0, 0.0, bad] if np.isinf(bad) else [bad] * 3
        q, _ = ref.project64(odd[0], w2cs[0], Ks[0])
        assert np.isnan(q[3, 5, 2])
        for path in ("ordered", "points4", "points1_align"):
            a = run_forward_warp(path, frames, None, odd, w2cs, Ks)
            b = run_forward_warp(path, frames, None, behind, w2cs, Ks)
            assert all(np.isfinite(x).all() for x in a[:3])
            if path == "ordered":
                assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
            else:
                res = ref.forward_warp(frames, None, behind, w2cs, Ks, b[3], BOUND_PATH[path])
                check_items(res, a[0], a[1], a[2], f"{bad} point {path}")


# ---------------------------------------------------------------------------------------------------------------------
# render_cache: items, groups, passes
# ---------------------------------------------------------------------------------------------------------------------
def cache_scene(B, Fs, N, F, H, W, seed):
    rng = np.random.RandomState(seed)
    pts, _, Ks = scene(H, W, B * Fs * N, 1.0, seed)
    points = pts.reshape(B, Fs, N, H, W, 3)
    images = rng.uniform(-1, 1, (B, Fs, N, 3, H, W)).astype(F32)
    masks = (rng.uniform(0, 1, (B, Fs, N, 1, H, W)) > 0.2).astype(F32)
    w2cs = np.stack([np.stack([target_camera((f * 7 + b) % 11) for f in range(F)]) for b in range(B)])
    Ks = np.broadcast_to(Ks[:1][None], (B, F, 3, 3)).copy()
    return points, images, masks, w2cs, Ks


def item_views(points, images, masks, w2cs, Ks):
    """The flattened (b, f, n) items of render_cache: per-item source arrays and cameras."""
    B, Fs, N = points.shape[:3]
    F = w2cs.shape[1]
    items = [(b, f, n) for b in range(B) for f in range(F) for n in range(N)]
    s = lambda f: 0 if Fs == 1 else f
    return (items, np.stack([points[b, s(f), n] for b, f, n in items]), np.stack([images[b, s(f), n] for b, f, n in items]),
            np.stack([masks[b, s(f), n, 0] for b, f, n in items]), np.stack([w2cs[b, f] for b, f, n in items]),
            np.stack([Ks[b, f] for b, f, n in items]))


CACHE_CASES = [  # B, Fs, N, F, H, W, max_items_per_pass
    (1, 1, 1, 1, 5, 13, 1), (1, 1, 3, 3, 8, 16, 4), (2, 1, 3, 3, 8, 12, 3), (2, 3, 2, 3, 5, 8, 4),
    (2, 3, 3, 3, 13, 16, 19), (1, 3, 1, 3, 3, 5, 3), (2, 1, 2, 1, 8, 16, 4), (1, 512, 1, 512, 4, 8, 4),
    (1, 1, 1, 513, 4, 8, 3), (1, 1, 3, 513, 4, 8, 4), (2, 1, 1, 513, 4, 8, 1540)]


@pytest.mark.parametrize("B,Fs,N,F,H,W,mpp", CACHE_CASES,
                         ids=[f"B={c[0]}-Fs={c[1]}-N={c[2]}-F={c[3]}-{c[4]}x{c[5]}-mpp={c[6]}" for c in CACHE_CASES])
@pytest.mark.parametrize("det", [False, True], ids=["atomic", "ordered"])
def test_render_cache_items(B, Fs, N, F, H, W, mpp, det):
    """Each chunk of two items (one shared log-depth max; with odd N a chunk spans two target cameras) equals
    forward_warp on the same pair: bitwise with the ordered splat, within the bound otherwise; and render_cache itself
    is within the bound of float64 on the positions forward_warp returns.  Fs = 1 with F <= 512 takes
    k_project_max_bcast, F = 513 (and Fs = F) the per-item k_project_max."""
    from gen3c_b200 import warp

    points, images, masks, w2cs, Ks = cache_scene(B, Fs, N, F, H, W, seed=B + 10 * N + F)
    with deterministic(det):
        pix, mk = warp.render_cache(cu(points), cu(images), cu(masks), cu(w2cs), cu(Ks), max_items_per_pass=mpp)
        dep, mk2 = warp.render_cache(cu(points), cu(images), cu(masks), cu(w2cs), cu(Ks), render_depth=True,
                                     max_items_per_pass=mpp)
    pix = pix.cpu().numpy().reshape(-1, 3, H, W)
    mk = mk.cpu().numpy().reshape(-1, H, W)
    dep = dep.cpu().numpy().reshape(-1, H, W)
    assert np.array_equal(mk, mk2.cpu().numpy().reshape(-1, H, W))
    items, P, I, M, Wc, Kc = item_views(points, images, masks, w2cs, Ks)
    n = len(items)
    path = "ordered" if det else ("points4" if W % 4 == 0 else "points1_w")
    worst = guard = 0.0
    for g0 in range(0, n, 2):
        s = slice(g0, min(g0 + 2, n))
        w, m, d, f = run_forward_warp(path, I[s], M[s], P[s], Wc[s], Kc[s])
        if det:
            assert np.array_equal(w, pix[s]) and np.array_equal(m, mk[s]) and np.array_equal(d, dep[s]), g0
        if g0 % 97 and g0 + 2 < n:        # float64 on a sample of chunks, always the first and the last
            continue
        res = ref.forward_warp(I[s], M[s], P[s], Wc[s], Kc[s], f, BOUND_PATH[path])
        wo, go = check_items(res, pix[s], mk[s], dep[s], f"render_cache chunk {g0} {path}")
        if not det:
            check_items(res, w, m, d, f"forward_warp chunk {g0} {path}")
        worst, guard = max(worst, wo), max(guard, go)
    print(f"\n[render-edges] render_cache B={B} Fs={Fs} N={N} F={F} mpp={mpp} det={det}: worst/bound {worst:.3g}")


def test_project_max_branch_by_camera_count():
    from gen3c_b200 import warp

    for F, want, avoid in ((512, "k_project_max_bcast", None), (513, "k_project_max", "k_project_max_bcast")):
        points, images, masks, w2cs, Ks = cache_scene(1, 1, 1, F, 4, 8, seed=F)
        args = [cu(x) for x in (points, images, masks, w2cs, Ks)]
        names = kernels_run(lambda: warp.render_cache(*args))
        assert any(want in x for x in names), (F, names)
        assert avoid is None or not any(avoid in x for x in names), (F, names)


def test_pass_sizes_and_camera_split_are_bitwise_equal():
    """Ordered splat: every pass size, including ones that leave a short last pass, gives the same bits; and a render
    of F = 513 targets (k_project_max) equals a render of the first 512 (k_project_max_bcast) plus one of the last."""
    from gen3c_b200 import warp

    B, Fs, N, F, H, W = 1, 1, 1, 513, 4, 8
    points, images, masks, w2cs, Ks = (cu(x) for x in cache_scene(B, Fs, N, F, H, W, seed=9))
    with deterministic():
        ref_pix, ref_mk = warp.render_cache(points, images, masks, w2cs, Ks, max_items_per_pass=4)
        for mpp in (1, 3, 5, 514):
            p, m = warp.render_cache(points, images, masks, w2cs, Ks, max_items_per_pass=mpp)
            assert torch.equal(p, ref_pix) and torch.equal(m, ref_mk), mpp
        a, am = warp.render_cache(points, images, masks, w2cs[:, :512].contiguous(), Ks[:, :512].contiguous())
        b, bm = warp.render_cache(points, images, masks, w2cs[:, 512:].contiguous(), Ks[:, 512:].contiguous())
    assert torch.equal(torch.cat([a, b], 1), ref_pix) and torch.equal(torch.cat([am, bm], 1), ref_mk)
    # the 6 x 4 items of test_cache_render_repeats_bitwise_whatever_the_pass_size, with pass sizes that do not divide
    points, images, masks, w2cs, Ks = (cu(x) for x in cache_scene(2, 3, 2, 3, 8, 16, seed=4))
    with deterministic():
        r0 = warp.render_cache(points, images, masks, w2cs, Ks, render_depth=True, max_items_per_pass=12)
        for mpp in (5, 7, 11, 13):
            r = warp.render_cache(points, images, masks, w2cs, Ks, render_depth=True, max_items_per_pass=mpp)
            assert torch.equal(r[0], r0[0]) and torch.equal(r[1], r0[1]), mpp


# ---------------------------------------------------------------------------------------------------------------------
# occlusion pass
# ---------------------------------------------------------------------------------------------------------------------
def test_occlusion_matches_oracle_off_multiple_of_4():
    """forward_warp(foreground_masking=True) at 37 x 50, b = 2, against warp_oracle: a pixel's removal may differ
    only where the float64 mesh depth lies within round-off of the splatted depth - 0.02."""
    from gen3c_b200 import warp

    h, w = 37, 50
    K = cases.intrinsics(h, w)
    depth = (2.9 + 0.35 * cases.smooth_depth(h, w)).astype(F32)
    depth[10:28, 14:34] = 1.2
    d = np.stack([depth, depth])[:, None]
    eye = np.stack([np.eye(4, dtype=F32)] * 2)
    Kb = np.stack([K, K])
    pts = warp_oracle.unproject_points(d, eye, Kb)
    bnd = ~warp_oracle.reliable_depth_mask_range_batch(d)[:, 0]
    tgt = np.stack([cases.look(0.06, -0.015, (0.12, 0.01, 0.03)), cases.look(-0.05, 0.02, (-0.1, 0.0, 0.05))])
    img = np.random.RandomState(0).uniform(-1, 1, (2, 3, h, w)).astype(F32)
    with deterministic():
        wk, mk, dk, fk = warp.forward_warp(cu(img), None, None, None, cu(tgt), None, cu(Kb), world_points1=cu(pts),
                                           foreground_masking=True, boundary_mask=cu(bnd))
    wk, mk, dk = (t.cpu().numpy() for t in (wk, mk, dk))
    wo, mo, do, _ = warp_oracle.forward_warp(img, None, pts, tgt, Kb, foreground_masking=True, boundary_mask=bnd)
    _, mplain, dplain, _ = warp_oracle.forward_warp(img, None, pts, tgt, Kb, render_depth=True)
    removed_o = (mplain[:, 0] > 0) & (mo[:, 0] == 0)
    removed_k = (mplain[:, 0] > 0) & (mk[:, 0] == 0)
    assert removed_o.mean() > 0.01
    # the mesh depth of the oracle, in float64 terms: within 1e-4 relative of the 0.02 threshold is round-off
    _, cam = warp_oracle.project_points(pts, tgt, Kb, return_cam_points=True)
    guard = np.zeros_like(removed_o)
    for i in range(2):
        verts, faces = warp_oracle.points_to_mesh(cam[i], bnd[i], (h // 4, w // 4))
        rays = warp_oracle.get_camera_rays(h, w, Kb[i])
        t = warp_oracle.ray_triangle_depth(np.zeros_like(rays), rays, verts, faces).reshape(h, w)
        mz = t.astype(np.float64) * rays[:, :, 2]
        guard[i] = (mz > 0) & (np.abs(mz + 0.02 - dplain[i]) <= 1e-4 * (1 + np.abs(dplain[i])))
    diff = removed_o != removed_k
    print(f"\n[render-edges] occlusion 37x50: removed {removed_o.mean():.4f}, guard {guard.mean():.4f}, "
          f"differ outside guard {int((diff & ~guard).sum())}")
    assert not (diff & ~guard).any()


def test_occlusion_passes_after_the_first():
    """render_cache with boundary masks and 66 items (F = 33, N = 2 at 16 x 24): the occlusion pass runs 64 + 2 items,
    and every item equals forward_warp(foreground_masking=True) on its chunk of two."""
    from gen3c_b200 import warp

    B, Fs, N, F, H, W = 1, 1, 2, 33, 16, 24
    points, images, masks, w2cs, Ks = cache_scene(B, Fs, N, F, H, W, seed=33)
    bnd = np.zeros((B, Fs, N, H, W), bool)
    bnd[..., 4:12, 6:18] = True
    bnd &= (np.random.RandomState(1).uniform(0, 1, bnd.shape) > 0.5)
    with deterministic():
        pix, mk = warp.render_cache(cu(points), cu(images), cu(masks), cu(w2cs), cu(Ks), boundary_masks=cu(bnd))
        pix, mk = pix.cpu().numpy().reshape(-1, 3, H, W), mk.cpu().numpy().reshape(-1, H, W)
        items, P, I, M, Wc, Kc = item_views(points, images, masks, w2cs, Ks)
        removed = 0
        for g0 in range(0, len(items), 2):
            s = slice(g0, g0 + 2)
            w, m, d, f = warp.forward_warp(cu(I[s]), cu(M[s][:, None]), None, None, cu(Wc[s]), None, cu(Kc[s]),
                                           world_points1=cu(P[s]), foreground_masking=True,
                                           boundary_mask=cu(np.stack([bnd[0, 0, n] for _, _, n in items[s]])))
            assert np.array_equal(w.cpu().numpy(), pix[s]) and np.array_equal(m.cpu().numpy()[:, 0], mk[s]), g0
            _, m0, _, _ = warp.forward_warp(cu(I[s]), cu(M[s][:, None]), None, None, cu(Wc[s]), None, cu(Kc[s]),
                                            world_points1=cu(P[s]))
            removed += int(((m0.cpu().numpy()[:, 0] > 0) & (mk[s] == 0)).sum()) if g0 >= 64 else 0
    assert removed > 0      # the items of the second pass do lose pixels to the occlusion test


# ---------------------------------------------------------------------------------------------------------------------
# unproject, reliability mask
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("is_depth", [True, False])
@pytest.mark.parametrize("with_mask", [False, True])
def test_unproject_points(is_depth, with_mask):
    from gen3c_b200 import warp

    rng = np.random.RandomState(int(is_depth) + 2 * int(with_mask))
    b, H, W = 2, 13, 37
    d = (rng.uniform(0.5, 30, (b, 1, H, W))).astype(F32)
    d[:, :, 2, :7] = 0
    d[:, :, 3, :7] = -2
    K = np.stack([cases.intrinsics(H, W), cases.intrinsics(H, W, f=11.0)])
    w2c = np.stack([cases.look(0.3, -0.2, (1.0, -2.0, 0.5)), cases.look(-1.0, 0.4, (10.0, 3.0, -4.0))])
    mask = (rng.uniform(0, 1, (b, 1, H, W)) > 0.3) if with_mask else None
    out = warp.unproject_points(cu(d), cu(w2c), cu(K), is_depth=is_depth,
                                mask=None if mask is None else cu(mask)).cpu().numpy()
    worst = 0.0
    for i in range(b):
        p, bnd, valid = ref.unproject64(d[i, 0], w2c[i], K[i], is_depth, None if mask is None else mask[i, 0])
        assert (out[i][~valid] == 0).all()
        worst = max(worst, float((np.abs(out[i] - p) / np.maximum(bnd, 1e-300)).max()))
    print(f"\n[render-edges] unproject is_depth={is_depth} mask={with_mask}: worst/bound {worst:.3g}")
    assert worst <= 1.0


@pytest.mark.parametrize("window", [1, 3, 5, 7])
@pytest.mark.parametrize("h,w", [(1, 1), (2, 3), (6, 5), (37, 45)])
def test_reliable_depth_mask(window, h, w):
    from gen3c_b200 import warp

    rng = np.random.RandomState(window * 100 + h)
    d = (2 + rng.uniform(0, 0.25, (3, 1, h, w))).astype(F32)
    d[rng.uniform(0, 1, d.shape) < 0.1] = 0
    out = warp.reliable_depth_mask_range_batch(cu(d), window_size=window, ratio_thresh=0.05).cpu().numpy()
    n_guard = 0
    for i in range(3):
        m, g = ref.reliable64(d[i, 0], window, 0.05)
        assert np.array_equal(out[i, 0][~g], m[~g]), i
        n_guard += int(g.sum())
    print(f"\n[render-edges] reliable window={window} {h}x{w}: guard {n_guard} of {d.size}")
    assert n_guard <= 0.02 * d.size + 1


# ---------------------------------------------------------------------------------------------------------------------
# depth alignment
# ---------------------------------------------------------------------------------------------------------------------
def align(depth, target, tmask, K, c2w, iters, lam=0.1, lr=1e-3):
    from gen3c_b200 import _lib

    H, W = depth.shape
    out = torch.full((H, W), -7.0, device="cuda")
    dt, tt, mt, kt, ct = cu(depth), cu(target), cu(tmask.astype(np.uint8)), cu(K), cu(c2w)
    _lib.check(_lib.load().g3c_align_depth_nonrigid(_lib.ptr(dt), _lib.ptr(tt), _lib.ptr(mt), _lib.ptr(kt),
                                                    _lib.ptr(ct), H, W, iters, lam, lr, _lib.ptr(out),
                                                    _lib.stream_ptr()), "g3c_align_depth_nonrigid")
    return out.cpu().numpy()


def align_case(H, W, mask_kind, seed):
    rng = np.random.RandomState(seed)
    d = (2 + rng.uniform(0, 1, (H, W))).astype(F32)
    t = (d * rng.uniform(0.95, 1.05, (H, W))).astype(F32)
    m = {"sparse": rng.uniform(0, 1, (H, W)) > 0.8, "empty": np.zeros((H, W), bool),
         "full": np.ones((H, W), bool)}[mask_kind]
    K = cases.intrinsics(H, W)
    c2w = cases.look(0.1, 0.05, (0.1, 0.0, 0.2))
    return d, t, m, K, c2w


@pytest.mark.parametrize("iters", [0, 1, 2, 5])
@pytest.mark.parametrize("H,W", [(37, 45), (9, 33), (8, 31)])
@pytest.mark.parametrize("mask_kind", ["sparse", "empty", "full"])
def test_align_depth_nonrigid(mask_kind, H, W, iters):
    """k_align_step on ragged 32 x 8 tiles (the halo's zero padding at a ragged edge); num_iters = 2 is the first case
    in which a tile's halo carries values that differ from the padding."""
    d, t, m, K, c2w = align_case(H, W, mask_kind, seed=H + iters)
    out = align(d, t, m, K, c2w, iters)
    r, tol, guard = ref.align64(d, t, m, K, c2w, iters)
    err = np.abs(out - r)
    worst = float((err / tol)[~guard].max())
    print(f"\n[render-edges] align {mask_kind} {H}x{W} iters={iters}: worst/tol {worst:.3g}, guard {guard.mean():.3f}"
          f" (in mask {guard[m].mean() if m.any() else 0:.3f})")
    assert worst <= 1.0
    if iters <= 1:
        assert not guard.any()
    if mask_kind == "sparse":          # data pixels (render_ref64.align64): few of them can be reached by a tie
        assert guard[m].mean() <= 0.2


@pytest.mark.parametrize("drop", ["m1", "m2"])
def test_align_negative_control(drop):
    """Dropping one Adam bias correction from the reference misses the tolerance on the kernel's output."""
    d, t, m, K, c2w = align_case(37, 45, "sparse", seed=1)
    for iters in (1, 2):
        out = align(d, t, m, K, c2w, iters)
        r, tol, guard = ref.align64(d, t, m, K, c2w, iters)
        bad, _, _ = ref.align64(d, t, m, K, c2w, iters, drop_bias=drop)
        assert (np.abs(out - r) / tol)[~guard].max() <= 1.0
        assert (np.abs(out - bad) / tol)[~guard].max() > 10.0


# ---------------------------------------------------------------------------------------------------------------------
# negative controls of the render bound on kernel output
# ---------------------------------------------------------------------------------------------------------------------
CONTROLS = {"crop_shift": dict(crop_shift=1), "per_item_max": dict(per_item_max=True),
            "ignore_mask": dict(ignore_mask=True), "swap_ne_sw": dict(swap_ne_sw=True), "no_soft_z": dict(soft_z=False)}


@pytest.mark.parametrize("control", list(CONTROLS))
@pytest.mark.parametrize("path", ["points4", "ordered"], ids=lambda p: f"path={p}")
def test_render_negative_controls(path, control):
    """Each deliberate error in the float64 reference misses the bar on this file's own kernel output: the crop
    shifted by a column, a per-item max instead of the shared one, the mask ignored, ne and sw swapped, no soft-z."""
    H, W, b = 24, 32, 2
    pts, w2cs, Ks = scene(H, W, b, 1.0, seed=21)
    pts[1] *= F32(0.5)
    rng = np.random.RandomState(21)
    frames = rng.uniform(-1, 1, (b, 3, H, W)).astype(F32)
    masks = (rng.uniform(0, 1, (b, H, W)) > 0.3).astype(F32) * rng.uniform(0.2, 1, (b, H, W)).astype(F32)
    w, m, d, f = run_forward_warp(path, frames, masks, pts, w2cs, Ks)
    good = ref.forward_warp(frames, masks, pts, w2cs, Ks, f, BOUND_PATH[path])
    check_items(good, w, m, d, f"control baseline {path}")
    bad = ref.forward_warp(frames, masks, pts, w2cs, Ks, f, BOUND_PATH[path], **CONTROLS[control])
    worst = 0.0
    for i in range(b):
        g = good[i]["guard"]
        flips = bool(((m[i] > 0) != (bad[i]["mask"] > 0))[~g].any())
        worst = max(worst, ref.excess(w[i], bad[i]["out"], good[i]["bound"], g), 1e9 if flips else 0.0)
    print(f"\n[render-edges] control {control} {path}: misses by {worst:.3g}x")
    assert worst > 10.0


# ---------------------------------------------------------------------------------------------------------------------
# error paths: G3C_EINVAL, nothing written
# ---------------------------------------------------------------------------------------------------------------------
def test_error_paths_write_nothing():
    from gen3c_b200 import _lib

    lib = _lib.load()
    st = _lib.stream_ptr()
    P = ctypes.c_void_p

    def fresh(*shape):
        return torch.full(shape, 7.0, device="cuda")

    def unchanged(*ts):
        torch.cuda.synchronize()
        return all(bool((t == 7.0).all()) for t in ts)

    H = W = 4
    ws = P()
    _lib.check(lib.g3c_render_create(H, W, 4, ctypes.byref(ws)))
    try:
        # B F N = 8193 items: 4097 groups of two exceed the 4096 maxima of the workspace
        F = 8193
        pts, img, w2c, K = fresh(F, H, W, 3), fresh(F, 3, H, W), fresh(F, 4, 4), fresh(F, 3, 3)
        pix, msk = fresh(F, 3, H, W), fresh(F, H, W)
        rc = lib.g3c_render_cache(ws, _lib.ptr(pts), _lib.ptr(img), None, _lib.ptr(w2c), _lib.ptr(K), 1, F, 1, F, 0,
                                  _lib.ptr(pix), _lib.ptr(msk), None, st)
        assert rc == -1 and unchanged(pix, msk)
        # src_frames not in {1, F}
        rc = lib.g3c_render_cache(ws, _lib.ptr(pts), _lib.ptr(img), None, _lib.ptr(w2c), _lib.ptr(K), 1, 3, 1, 2, 0,
                                  _lib.ptr(pix), _lib.ptr(msk), None, st)
        assert rc == -1 and unchanged(pix, msk)
        # C = 4
        out, m2, fl = fresh(1, 4, H, W), fresh(1, H, W), fresh(1, 2, H, W)
        rc = lib.g3c_forward_warp(ws, _lib.ptr(pts), _lib.ptr(fresh(1, 4, H, W)), None, _lib.ptr(w2c), _lib.ptr(K), 1, 4,
                                  0, _lib.ptr(out), _lib.ptr(m2), None, _lib.ptr(fl), st)
        assert rc == -1 and unchanged(out, m2, fl)
        # occlusion on frames under 8 rows
        bm = torch.ones(1, 7, 16, device="cuda", dtype=torch.uint8)
        o3, m3, d3 = fresh(1, 3, 7, 16), fresh(1, 7, 16), fresh(1, 7, 16)
        rc = lib.g3c_foreground_occlusion(_lib.ptr(fresh(1, 7, 16, 3)), _lib.ptr(bm), _lib.ptr(w2c), _lib.ptr(K), 1, 3,
                                          7, 16, _lib.ptr(o3), _lib.ptr(m3), _lib.ptr(d3), st)
        assert rc == -1 and unchanged(o3, m3, d3)
        rc = lib.g3c_render_cache_occlusion(_lib.ptr(fresh(1, 7, 16, 3)), _lib.ptr(bm), _lib.ptr(w2c), _lib.ptr(K), 1, 1,
                                            1, 1, _lib.ptr(o3), _lib.ptr(m3), _lib.ptr(d3), 7, 16, st)
        assert rc == -1 and unchanged(o3, m3, d3)
    finally:
        lib.g3c_render_destroy(ws)
