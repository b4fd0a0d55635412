"""GPU parity for Path R: the CUDA render (through the C ABI) against the numpy oracle and the golden
vectors minted from the reference.  Tolerances: integer indices bit-exact; float outputs fp32 round-off
amplified by the soft-z weights (atol 2e-3 on [-1,1] images away from coverage edges, mask flips bounded)."""
import os

import numpy as np
import pytest
import torch

from oracle import cases, golden, warp_oracle

pytestmark = pytest.mark.gpu


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def close_frac(a, b, atol):
    return float((np.abs(a - b) <= atol).mean())


@pytest.mark.parametrize("name", ["R1", "R2", "R3", "R4", "R5", "R6"])
def test_forward_warp_matches_reference_golden(name, golden_dir):
    from gen3c_b200 import warp

    g = golden.load(golden_dir, f"warp_{name}")
    c = cases.warp_case(name)
    pts = warp.unproject_points(cu(c["depth"]), cu(c["w2c_src"]), cu(c["K"]))
    np.testing.assert_allclose(pts.cpu().numpy(), g["points"], atol=5e-5, rtol=1e-5)
    # same world points as the reference -> isolates project + splat
    w, m, d, f = warp.forward_warp(cu(c["image"]), None if c["mask"] is None else cu(c["mask"]), None, None,
                                   cu(c["w2c_tgt"]), cu(c["K"]), cu(c["K"]), render_depth=True,
                                   world_points1=cu(g["points"]))
    torch.cuda.synchronize()
    w, m, d, f = (t.cpu().numpy() for t in (w, m, d, f))
    np.testing.assert_allclose(f, g["flow"], atol=2e-3)  # flow in pixels; fp32 projection order differs
    assert (m != g["mask"]).mean() < 2e-3                # coverage flips only at splat boundaries
    same = (m == g["mask"]) & (g["mask"] > 0)
    sel = np.broadcast_to(same, w.shape)
    assert close_frac(w[sel], g["warped"][sel], 2e-3) > 0.999
    assert np.abs(w[sel] - g["warped"][sel]).mean() < 1e-4
    assert close_frac(d[same[:, 0]], g["depth"][same[:, 0]], 1e-3) > 0.999


def test_forward_warp_width_not_multiple_of_4():
    """A frame with W % 4 != 0 takes the one-pixel-per-thread splat kernel (k_splat_points), not the 4-pixel one."""
    from gen3c_b200 import warp

    c = cases.warp_case("R6")
    depth, image = (np.ascontiguousarray(c[k][..., :126]) for k in ("depth", "image"))
    pts = warp.unproject_points(cu(depth), cu(c["w2c_src"]), cu(c["K"]))
    w, m, d, f = warp.forward_warp(cu(image), None, None, None, cu(c["w2c_tgt"]), cu(c["K"]), cu(c["K"]),
                                   render_depth=True, world_points1=pts)
    torch.cuda.synchronize()
    w, m, d, f = (t.cpu().numpy() for t in (w, m, d, f))
    wo, mo, do, fo = warp_oracle.forward_warp(image, None, pts.cpu().numpy(), c["w2c_tgt"], c["K"], render_depth=True)
    np.testing.assert_allclose(f, fo, atol=2e-3)
    assert (m != mo).mean() < 2e-3
    same = (m == mo) & (mo > 0)
    sel = np.broadcast_to(same, w.shape)
    assert close_frac(w[sel], wo[sel], 2e-3) > 0.999
    assert np.abs(w[sel] - wo[sel]).mean() < 1e-4
    assert close_frac(d[same[:, 0]], do[same[:, 0]], 1e-3) > 0.999


@pytest.mark.parametrize("name", ["R2", "R4", "R6"])
def test_splat_indices_bit_exact(name, golden_dir):
    """Integer work: floor/ceil/clamp destination indices on the reference's own coordinates."""
    from gen3c_b200 import warp

    g = golden.load(golden_dir, f"warp_{name}")
    idx = warp.splat_indices(cu(g["flow"])).cpu().numpy()
    assert np.array_equal(idx[:, 0], g["floor"][:, 0]) and np.array_equal(idx[:, 1], g["floor"][:, 1])
    assert np.array_equal(idx[:, 2], g["ceil"][:, 0]) and np.array_equal(idx[:, 3], g["ceil"][:, 1])


def test_bilinear_splatting_on_shared_coordinates(golden_dir):
    """Splat alone on the reference's flow/depth: only atomics order and exp/log ulps differ."""
    from gen3c_b200 import warp

    g = golden.load(golden_dir, "warp_R6")
    c = cases.warp_case("R6")
    z = warp_oracle.project_points(g["points"], c["w2c_tgt"], c["K"])[:, :, :, 2][:, None]
    mask = (z > 0).astype(np.float32)
    ref, rmask = warp_oracle.bilinear_splatting(c["image"], mask, z, g["flow"], is_image=True)
    out, omask = warp.bilinear_splatting(cu(c["image"]), cu(mask), cu(z), cu(g["flow"]), is_image=True)
    out, omask = out.cpu().numpy(), omask.cpu().numpy()
    assert np.array_equal(omask, rmask)
    np.testing.assert_allclose(out, ref, atol=2e-4)


def test_degenerate_integer_coordinates():
    from gen3c_b200 import warp

    flow = torch.full((1, 2, 8, 8), 2.0, device="cuda")
    img = torch.rand(1, 3, 8, 8, device="cuda") * 2 - 1
    out, mask = warp.bilinear_splatting(img, None, torch.ones(1, 1, 8, 8, device="cuda"), flow, is_image=True)
    torch.testing.assert_close(out[:, :, 2:, 2:], img[:, :, :-2, :-2], atol=1e-6, rtol=0)
    assert float(mask[:, :, :2].max()) == 0 and float(mask[:, :, :, :2].max()) == 0
    assert float(out[:, :, :2].max()) == -1.0  # unknown pixels of an image are filled with -1


def test_render_cache_matches_reference_golden(golden_dir):
    """Cache3D render, N=2 buffers, F=3 targets, chunk-of-2 max coupling (cache_3d.py:175-223)."""
    from gen3c_b200 import warp

    g = golden.load(golden_dir, "warp_cache")
    c = cases.warp_case("R3")
    F = 3
    w2cs = cases.pan_trajectory(F, 0.1)[None]
    Ks = np.tile(c["K"][:1], (F, 1, 1))[None]
    pix, msk = warp.render_cache(cu(g["points"]), cu(c["image"][None, None]), cu(g["cache_mask"]), cu(w2cs), cu(Ks))
    pix, msk = pix.cpu().numpy(), msk.cpu().numpy()
    assert (msk != g["masks"]).mean() < 2e-3
    same = np.broadcast_to((msk == g["masks"]) & (g["masks"] > 0), pix.shape)
    assert close_frac(pix[same], g["pixels"][same], 2e-3) > 0.999
    rel = warp.reliable_depth_mask_range_batch(cu(c["depth"].reshape(-1, 1, 96, 128)), ratio_thresh=0.05)
    assert (rel.cpu().numpy() != g["reliable"]).mean() < 1e-4


def test_full_size_identity_roundtrip():
    """BASELINE size (704x1280): unproject -> identity camera warp reproduces the image (size-independent
    property, no oracle needed), and a chunk rendered through render_cache equals forward_warp on the pair."""
    from gen3c_b200 import warp

    h, w = 704, 1280
    depth = cu(cases.smooth_depth(h, w)[None, None])
    K = cu(cases.intrinsics(h, w)[None])
    eye = torch.eye(4, device="cuda")[None]
    g = torch.Generator(device="cuda").manual_seed(0)
    img = torch.rand(1, 3, h, w, device="cuda", generator=g) * 2 - 1
    pts = warp.unproject_points(depth, eye, K)
    out, mask, dep, _ = warp.forward_warp(img, None, None, None, eye, K, K, render_depth=True, world_points1=pts)
    assert float(mask.min()) == 1.0
    # identity warp = integer target coordinates +- 1 ulp (ulp of 1280 is 1.2e-4): a sub-pixel sliver of the
    # neighbour leaks in, amplified by the soft-z weight; the numpy oracle shows 2.4e-4 at 256x256.
    assert float((out - img).abs().max()) <= 2e-3
    assert float((out - img).abs().mean()) <= 1e-4
    assert float((dep - depth[:, 0]).abs().max()) <= 1e-3
    w2cs = cu(cases.pan_trajectory(2, 0.05))[None]
    pix, msk = warp.render_cache(pts[None, None], img[None, None], None, w2cs, K[None].expand(1, 2, 3, 3).contiguous())
    pair, pmask, _, _ = warp.forward_warp(img.expand(2, -1, -1, -1).contiguous(), None, None, None, w2cs[0],
                                          K.expand(2, 3, 3).contiguous(), None, world_points1=pts.expand(2, -1, -1, -1).contiguous())
    assert torch.equal(msk[0, :, 0], pmask)
    assert float((pix[0, :, 0] - pair).abs().max()) <= 1e-5


def test_foreground_masking_matches_reference_golden(golden_dir):
    """forward_warp(foreground_masking=True): the native occlusion pass against the golden minted from the reference's
    own forward_warp (tests/golden/warp_R7_foreground.npz).  Occlusion decisions may flip only on knife-edge pixels
    (mesh depth within float round-off of `splatted depth - 0.02`)."""
    from gen3c_b200 import warp

    g = golden.load(golden_dir, "warp_R7_foreground")
    c = cases.foreground_case()
    w, m, d, _ = warp.forward_warp(cu(c["image"]), None, None, None, cu(c["w2c_tgt"]), cu(c["K"]), cu(c["K"]),
                                   world_points1=cu(g["points"]), foreground_masking=True, boundary_mask=cu(g["boundary"]))
    torch.cuda.synchronize()
    w, m, d = (t.cpu().numpy() for t in (w, m, d))
    occluded_ref = (g["mask_plain"] > 0) & (g["mask"] == 0)
    occluded = (g["mask_plain"] > 0) & (m == 0)
    assert occluded_ref.mean() > 0.02
    assert (occluded != occluded_ref).mean() < 2e-3
    same = (m == g["mask"])
    sel = np.broadcast_to(same, w.shape)
    assert close_frac(w[sel], g["warped"][sel], 2e-3) > 0.999
    assert close_frac(d[same[:, 0]], g["depth"][same[:, 0]], 1e-3) > 0.999


def test_foreground_masking_full_size_properties():
    """704x1280 (BASELINE frame size; the brute-force oracle would need 1e11 ray/triangle tests): a near box in front of a
    smooth background, camera shifted.  Size-independent properties of the occlusion pass: it only ever REMOVES pixels;
    every removed pixel was background (splatted depth well behind the box); everything else is bit-identical to the
    plain warp; and the cache-level path (g3c_render_cache + g3c_render_cache_occlusion through Cache3D_Base) returns
    exactly what forward_warp(foreground_masking=True) returns for the same frame."""
    from gen3c_b200 import warp
    from gen3c_b200.cache_3d import Cache3D_Base

    h, w = 704, 1280
    depth = (2.9 + 0.35 * cases.smooth_depth(h, w)).astype(np.float32)
    depth[220:520, 440:840] = 1.2
    g = torch.Generator(device="cuda").manual_seed(0)
    img = torch.rand(1, 3, h, w, device="cuda", generator=g) * 2 - 1
    K = cu(cases.intrinsics(h, w)[None])
    eye = torch.eye(4, device="cuda")[None]
    tgt = cu(cases.look(0.06, -0.015, (0.12, 0.01, 0.03))[None])
    d = cu(depth[None, None])
    pts = warp.unproject_points(d, eye, K)
    boundary = ~warp.reliable_depth_mask_range_batch(d)[:, 0]
    assert 1e-4 < float(boundary.float().mean()) < 0.05
    w0, m0, z0, _ = warp.forward_warp(img, None, None, None, tgt, K, K, render_depth=True, world_points1=pts)
    w1, m1, z1, _ = warp.forward_warp(img, None, None, None, tgt, K, K, world_points1=pts, foreground_masking=True,
                                      boundary_mask=boundary)
    removed = (m0 > 0) & (m1 == 0)
    assert bool(((m1 > 0) <= (m0 > 0)).all())                     # never adds coverage
    assert float(removed.float().mean()) > 1e-3                   # the box edge does occlude something
    assert float(z0[removed[:, 0]].min()) > 1.2 + 0.02            # only background goes
    keep = ~removed
    # (two separate splats: equal up to the order of their float atomics)
    assert float((w1 - w0)[keep.expand_as(w1)].abs().max()) < 1e-4 and float((z1 - z0)[keep[:, 0]].abs().max()) < 1e-4
    assert float(w1[removed.expand_as(w1)].max()) == -1.0 and float(z1[removed[:, 0]].max()) == 0.0
    cache = Cache3D_Base(input_image=img, input_depth=d, input_w2c=eye, input_intrinsics=K, foreground_masking=True)
    pix, msk = cache.render_cache(tgt[None], K[None])
    assert float((msk[0, 0] != m1[0][None]).float().mean()) < 1e-5 and float((pix[0, 0, 0] - w1[0]).abs().max()) < 1e-4


def test_error_behaviour():
    from gen3c_b200 import warp

    img = torch.zeros(1, 3, 8, 8, device="cuda")
    with pytest.raises(AssertionError):
        warp.forward_warp(img, None, None, None, torch.eye(4, device="cuda")[None], None, None,
                          world_points1=torch.zeros(1, 8, 8, 3, device="cuda"))
    with pytest.raises(AssertionError):   # foreground_masking without a boundary mask (reference :286)
        warp.forward_warp(img, None, None, None, torch.eye(4, device="cuda")[None], None,
                          torch.eye(3, device="cuda")[None], world_points1=torch.zeros(1, 8, 8, 3, device="cuda"),
                          foreground_masking=True)
    with pytest.raises(NotImplementedError):
        warp.forward_warp(img, None, None, None, torch.eye(4, device="cuda")[None], None,
                          torch.eye(3, device="cuda")[None], world_points1=torch.zeros(1, 8, 8, 3, device="cuda"),
                          cameraray_filtering=True)
    with pytest.raises(AssertionError):
        warp.reliable_depth_mask_range_batch(torch.ones(1, 1, 8, 8, device="cuda"), window_size=4)
