"""Path R under torch.use_deterministic_algorithms(True): the ordered, atomic-free splat (g3c_render_set_deterministic).

The contract pinned here: every destination texel sums its contributions sequentially in fp32 from 0, corner-major
(nw, sw, ne, se), then in ascending source pixel -- the order of np.add.at in oracle/warp_oracle.py and of the
reference's index_put_(accumulate=True) under the flag.  With depth == 0 the weights are exact in numpy and on the
device, so the native splat must equal the oracle bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import cases, golden, warp_oracle

from . import test_cache_gpu, test_warp_gpu

pytestmark = pytest.mark.gpu

F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture
def deterministic():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    # warn_only: torch ops outside this library that have no deterministic implementation warn instead of failing
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _oracle_reversed(frame, mask, depth, flow, is_image):
    """warp_oracle.bilinear_splatting with the sources of every corner visited in DESCENDING order (negative control)."""
    b, c, h, w = frame.shape
    pos, fl, ce = warp_oracle.splat_indices(flow)
    flf, cef = fl.astype(F32), ce.astype(F32)
    one = F32(1)
    w_nw = (one - (pos[:, 1:2] - flf[:, 1:2])) * (one - (pos[:, 0:1] - flf[:, 0:1]))
    w_sw = (one - (cef[:, 1:2] - pos[:, 1:2])) * (one - (pos[:, 0:1] - flf[:, 0:1]))
    w_ne = (one - (pos[:, 1:2] - flf[:, 1:2])) * (one - (cef[:, 0:1] - pos[:, 0:1]))
    w_se = (one - (cef[:, 1:2] - pos[:, 1:2])) * (one - (cef[:, 0:1] - pos[:, 0:1]))
    logd = np.log1p(np.maximum(depth, F32(0))).astype(F32)
    dw = np.exp(np.minimum(logd / (logd.max() + F32(1e-7)) * F32(50), F32(80))).astype(F32) + F32(1e-7)
    acc = np.zeros((b, h + 2, w + 2, c), F32)
    wsum = np.zeros((b, h + 2, w + 2, 1), F32)
    bidx = np.broadcast_to(np.arange(b)[:, None, None], (b, h, w)).reshape(-1)[::-1]
    frame_cl = np.moveaxis(frame, 1, 3).reshape(-1, c)[::-1]
    for wt, yy, xx in ((w_nw, fl[:, 1], fl[:, 0]), (w_sw, ce[:, 1], fl[:, 0]),
                       (w_ne, fl[:, 1], ce[:, 0]), (w_se, ce[:, 1], ce[:, 0])):
        wgt = np.moveaxis((wt * mask / dw).astype(F32), 1, 3).reshape(-1, 1)[::-1]
        idx = (bidx, yy.reshape(-1)[::-1], xx.reshape(-1)[::-1])
        np.add.at(acc, idx, (frame_cl * wgt).astype(F32))
        np.add.at(wsum, idx, wgt)
    acc = np.moveaxis(acc, 3, 1)[:, :, 1:-1, 1:-1]
    ws = np.moveaxis(wsum, 3, 1)[:, :, 1:-1, 1:-1]
    hit = ws > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        out = np.where(hit, acc / ws, F32(-1 if is_image else 0)).astype(F32)
    return (np.clip(out, -1, 1) if is_image else out), hit.astype(F32)


def _jitter_and_dolly_flow(rng, b, h, w):
    """Sub-pixel jitter everywhere; the central h/2 x w/2 region contracts 8x towards its centre (a dolly-out), so its
    texels receive tens of records each."""
    flow = rng.uniform(-0.6, 0.6, (b, 2, h, w)).astype(F32)
    ys, xs = np.mgrid[0:h, 0:w].astype(F32)
    cy, cx = F32(h / 2 + 0.3), F32(w / 2 - 0.2)
    reg = (np.abs(ys - cy) < h / 4) & (np.abs(xs - cx) < w / 4)
    flow[:, 0][:, reg] = ((cx + (xs - cx) / F32(8)) - xs)[reg] + rng.uniform(-0.2, 0.2, (b, int(reg.sum())))
    flow[:, 1][:, reg] = ((cy + (ys - cy) / F32(8)) - ys)[reg] + rng.uniform(-0.2, 0.2, (b, int(reg.sum())))
    return flow.astype(F32)


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("is_image", [False, True])
def test_splat_order_is_the_reference_order_bit_for_bit(deterministic, C, is_image):
    from gen3c_b200 import warp

    rng = np.random.RandomState(10 * C + int(is_image))
    b, h, w = 2, 96, 128
    frame = rng.uniform(-1, 1, (b, C, h, w)).astype(F32)
    mask = rng.uniform(0, 1, (b, 1, h, w)).astype(F32)
    depth = np.zeros((b, 1, h, w), F32)
    flow = _jitter_and_dolly_flow(rng, b, h, w)
    ref, rmask = warp_oracle.bilinear_splatting(frame, mask, depth, flow, is_image=is_image)
    out, omask = warp.bilinear_splatting(cu(frame), cu(mask), cu(depth), cu(flow), is_image=is_image)
    assert np.array_equal(omask.cpu().numpy(), rmask)
    assert np.array_equal(out.cpu().numpy(), ref)
    # the test can fail: summing the same records in another order changes the result
    rev, _ = _oracle_reversed(frame, mask, depth, flow, is_image)
    assert not np.array_equal(rev, ref)


def _concentrated_flow(h, w, py, px):
    grid = warp_oracle.create_grid(1, h, w)
    return (np.array([px, py], F32).reshape(1, 2, 1, 1) - grid).astype(F32)


def test_concentrated_splat_matches_oracle(deterministic):
    """Every source of a 256 x 256 frame lands on one sub-pixel point: 4 texels with 65 536 records each."""
    from gen3c_b200 import warp

    rng = np.random.RandomState(3)
    h = w = 256
    frame = rng.uniform(-1, 1, (1, 3, h, w)).astype(F32)
    mask = rng.uniform(0.1, 1, (1, 1, h, w)).astype(F32)
    depth = np.zeros((1, 1, h, w), F32)
    flow = _concentrated_flow(h, w, 100.3, 57.6)
    ref, rmask = warp_oracle.bilinear_splatting(frame, mask, depth, flow, is_image=True)
    out, omask = warp.bilinear_splatting(cu(frame), cu(mask), cu(depth), cu(flow), is_image=True)
    assert rmask.sum() == 4
    assert np.array_equal(omask.cpu().numpy(), rmask)
    assert np.array_equal(out.cpu().numpy(), ref)


def test_concentrated_splat_full_size_repeats(deterministic):
    from gen3c_b200 import warp

    h, w = 704, 1280
    g = torch.Generator(device="cuda").manual_seed(4)
    frame = torch.rand(1, 3, h, w, device="cuda", generator=g) * 2 - 1
    depth = torch.rand(1, 1, h, w, device="cuda", generator=g) * 3
    flow = cu(_concentrated_flow(h, w, 351.25, 640.7))
    a = warp.bilinear_splatting(frame, None, depth, flow, is_image=True)
    b = warp.bilinear_splatting(frame, None, depth, flow, is_image=True)
    assert float(a[1].sum()) == 4.0
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


GOLDEN_CHECKS = ([(test_warp_gpu.test_forward_warp_matches_reference_golden, {"name": n})
                  for n in ("R1", "R2", "R3", "R4", "R5", "R6")] +
                 [(test_warp_gpu.test_bilinear_splatting_on_shared_coordinates, {}),
                  (test_warp_gpu.test_degenerate_integer_coordinates, {}),
                  (test_warp_gpu.test_render_cache_matches_reference_golden, {}),
                  (test_warp_gpu.test_full_size_identity_roundtrip, {}),
                  (test_warp_gpu.test_foreground_masking_matches_reference_golden, {}),
                  (test_warp_gpu.test_foreground_masking_full_size_properties, {}),
                  (test_cache_gpu.test_buffer_ring_of_two_matches_reference, {}),
                  (test_cache_gpu.test_buffer_noise_branch, {}),
                  (test_cache_gpu.test_update_cache_with_depth_alignment_matches_reference, {"method": "rigid"}),
                  (test_cache_gpu.test_update_cache_with_depth_alignment_matches_reference, {"method": "non_rigid"}),
                  (test_cache_gpu.test_buffer_selector_and_cache4d_match_reference, {}),
                  (test_cache_gpu.test_unproject_ray_depth_and_forward_warp_from_depth, {})])


@pytest.mark.parametrize("check,kw", GOLDEN_CHECKS,
                         ids=[f.__name__ + "".join(f"-{v}" for v in kw.values()) for f, kw in GOLDEN_CHECKS])
def test_golden_checks_hold_under_the_flag(deterministic, golden_dir, check, kw):
    """The existing golden checks, unchanged tolerances, with the ordered splat."""
    import inspect

    params = inspect.signature(check).parameters
    if "golden_dir" in params:
        kw = dict(kw, golden_dir=golden_dir)
    if "g" in params:
        kw = dict(kw, g=golden.load(golden_dir, "warp_cache_classes"))
    check(**kw)


def _full_size_scene():
    from gen3c_b200 import warp

    h, w = 704, 1280
    K = cu(cases.intrinsics(h, w)[None])
    g = torch.Generator(device="cuda").manual_seed(7)
    pts, imgs, bms = [], [], []
    for n, src in enumerate((np.eye(4, dtype=F32), cases.look(0.04, 0.0, (0.05, 0.0, 0.0)))):
        depth = (2.9 + 0.35 * cases.smooth_depth(h, w)).astype(F32)
        depth[200 + 40 * n:500, 400:800 + 40 * n] = 1.3
        d = cu(depth[None, None])
        s = cu(src[None])
        pts.append(warp.unproject_points(d, s, K))
        imgs.append(torch.rand(1, 3, h, w, device="cuda", generator=g) * 2 - 1)
        bms.append(~warp.reliable_depth_mask_range_batch(d)[:, 0])
    pan = cases.pan_trajectory(6, 0.2)
    dolly = np.stack([cases.look(0.0, 0.0, (0.0, 0.0, 0.4 * k)) for k in range(1, 7)])  # camera backs away
    w2cs = cu(np.concatenate([pan, dolly]).astype(F32))[None]
    Ks = K[None].expand(1, 12, 3, 3).contiguous()
    points = torch.stack([p[0] for p in pts])[None, None]        # (1, 1, 2, H, W, 3)
    images = torch.stack([i[0] for i in imgs])[None, None]       # (1, 1, 2, 3, H, W)
    masks = (torch.rand(1, 1, 2, 1, h, w, device="cuda", generator=g) > 0.05).float()
    boundary = torch.stack([m[0] for m in bms])[None, None]      # (1, 1, 2, H, W)
    return points, images, masks, w2cs, Ks, boundary


def test_cache_render_repeats_bitwise_whatever_the_pass_size(deterministic):
    from gen3c_b200 import warp

    points, images, masks, w2cs, Ks, boundary = _full_size_scene()

    def render(m):
        return warp.render_cache(points, images, masks, w2cs, Ks, render_depth=True, max_items_per_pass=m,
                                 boundary_masks=boundary)

    def pixels(m):  # render_depth=True returns the depth; the pixels of the same call are rendered alongside
        return warp.render_cache(points, images, masks, w2cs, Ks, max_items_per_pass=m, boundary_masks=boundary)

    d0, m0 = render(4)
    p0, _ = pixels(4)
    assert 0.05 < float(m0.mean()) < 0.99
    for m in (4, 4, 1, 2):
        d, mk = render(m)
        p, _ = pixels(m)
        assert torch.equal(d, d0) and torch.equal(mk, m0) and torch.equal(p, p0), m
    # forward_warp on items (2k, 2k + 1) -- the two buffers of target k, one log-depth max -- is the same render
    for k in (0, 5, 6, 11):
        wp, wm, wd, _ = warp.forward_warp(images[0, 0], masks[0, 0], None, None, w2cs[0, k:k + 1].expand(2, 4, 4).contiguous(),
                                          None, Ks[0, k:k + 1].expand(2, 3, 3).contiguous(), world_points1=points[0, 0],
                                          render_depth=True, foreground_masking=True, boundary_mask=boundary[0, 0])
        assert torch.equal(wp, p0[0, k]) and torch.equal(wm, m0[0, k]) and torch.equal(wd, d0[0, k]), k


_E2E = r"""
import pathlib, sys
import numpy as np, torch
torch.use_deterministic_algorithms(True, warn_only=True)
from tests.test_entry_point_gpu import _args, _pipeline
out = pathlib.Path(sys.argv[1])
for name, over in (("fg", dict(foreground_masking=True, save_buffer=True)),
                   ("two_chunks", dict(num_video_frames=241, trajectory="clockwise"))):
    (out / name).mkdir()
    m, args = _args(out / name, **over)
    (_, video), = m.demo(args, pipeline=_pipeline(args))
    np.save(out / f"{name}.npy", video)
"""


def test_end_to_end_generation_is_bitwise_reproducible(tmp_path):
    """Two separate processes, same seed, the flag on, the arguments of test_entry_point_gpu.py: the single-image demo
    with foreground masking, and the two-chunk autoregressive run (update_cache with depth alignment), each save the
    same video bit for bit."""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8",
               PYTHONPATH=os.pathsep.join([ROOT] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    videos = []
    for r in range(2):
        out = tmp_path / f"run{r}"
        out.mkdir()
        subprocess.run([sys.executable, "-c", _E2E, str(out)], cwd=ROOT, env=env, check=True, timeout=900)
        videos.append({k: np.load(out / f"{k}.npy") for k in ("fg", "two_chunks")})
    assert videos[0]["fg"].shape == (121, 128, 512, 3) and videos[0]["two_chunks"].shape == (241, 128, 256, 3)
    for k in ("fg", "two_chunks"):
        assert np.array_equal(videos[0][k], videos[1][k]), k
