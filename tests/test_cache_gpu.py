"""GPU parity of the cache classes (gen3c_b200/cache_3d.py, camera_utils.align_depth, the is_depth=False and depth1
branches of the warp operators) against goldens minted from the reference's own classes on CPU
(tests/golden/warp_cache_classes.npz).  Float tolerances as in test_warp_gpu.py: fp32 round-off amplified by the soft-z
weights (2e-3 on [-1,1] images for >= 99.9 % of the commonly covered pixels, < 0.2 % coverage flips)."""
import os

import numpy as np
import pytest
import torch

from oracle import cases, golden

pytestmark = pytest.mark.gpu


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def g(golden_dir):
    return golden.load(golden_dir, "warp_cache_classes")


def same_render(pix, msk, ref_pix, ref_msk, atol=2e-3, flips=2e-3, frac=0.999):
    pix, msk = pix.cpu().numpy(), msk.cpu().numpy()
    assert pix.shape == ref_pix.shape and msk.shape == ref_msk.shape
    assert (msk != ref_msk).mean() < flips, (msk != ref_msk).mean()
    both = (msk == ref_msk) & (ref_msk > 0)
    sel = np.broadcast_to(both, pix.shape) if pix.ndim == both.ndim else both[:, :, :, 0]
    assert (np.abs(pix[sel] - ref_pix[sel]) <= atol).mean() > frac


def _targets():
    c3 = cases.warp_case("R3")
    K = cu(c3["K"][:1])
    F = 2
    return c3, K, cu(cases.pan_trajectory(F, 0.08))[None], K[None].expand(1, F, 3, 3).contiguous()


def _buffer(c3, K, **kw):
    from gen3c_b200.cache_3d import Cache3D_Buffer

    return Cache3D_Buffer(frame_buffer_max=2, noise_aug_strength=0, generator=None, input_image=cu(c3["image"][:1]),
                          input_depth=cu(c3["depth"][:1]), input_w2c=cu(c3["w2c_src"][:1]), input_intrinsics=K,
                          filter_points_threshold=0.05, **kw)


def test_buffer_ring_of_two_matches_reference(g):
    """Cache3D_Buffer: construct (['B','C','H','W'] canonicalisation, reliability mask), render, append a second frame,
    overwrite slot 0 when the ring is full, depth render — reference cache_3d.py:239-343."""
    c3, K, w2cs, Ks = _targets()
    c6 = cases.warp_case("R6")
    cache = _buffer(c3, K)
    assert cache.input_frame_count() == 1 and cache.input_image.shape == (1, 1, 1, 1, 3, 96, 128)
    same_render(*cache.render_cache(w2cs, Ks), g["buf_p0"], g["buf_m0"])
    cache.update_cache(cu(c3["image"][1:2]), cu(c3["depth"][1:2]), cu(g["buf_new_w2c"]), new_intrinsics=K,
                       depth_alignment=False)
    assert cache.input_image.shape[2] == 2
    same_render(*cache.render_cache(w2cs, Ks), g["buf_p1"], g["buf_m1"])
    cache.update_cache(cu(c6["image"]), cu(c6["depth"]), cu(g["buf_new_w2c2"]), new_intrinsics=K, depth_alignment=False)
    assert cache.input_image.shape[2] == 2
    same_render(*cache.render_cache(w2cs, Ks), g["buf_p2"], g["buf_m2"])
    dep, dm = cache.render_cache(w2cs, Ks, render_depth=True)
    same_render(dep, dm, g["buf_d2"], g["buf_m2"], atol=1e-3)
    with pytest.raises(AssertionError):
        cache.render_cache(w2cs, Ks, start_frame_idx=1)


def test_buffer_noise_branch():
    """noise_aug_strength > 0: the newest buffer (slot 0) is clean... of N = 2 slots, slot 0 gets (N-1-0) = 1 x strength,
    slot 1 gets 0 (reference :336-343: arange(N-1, -1, -1)); the draw uses the caller's generator."""
    from gen3c_b200.cache_3d import Cache3D_Buffer

    c3, K, w2cs, Ks = _targets()
    imgs = cu(np.stack([c3["image"][0], c3["image"][1]])[None])
    deps = cu(np.stack([c3["depth"][0], c3["depth"][1]])[None])
    src = cu(np.stack([c3["w2c_src"][0], c3["w2c_src"][1]])[None])
    kw = dict(input_image=imgs, input_depth=deps, input_w2c=src, input_intrinsics=K[None].expand(1, 2, 3, 3).contiguous(),
              input_format=["B", "N", "C", "H", "W"], frame_buffer_max=2)
    clean = Cache3D_Buffer(noise_aug_strength=0.0, generator=torch.Generator(device="cuda").manual_seed(3), **kw)
    noisy = Cache3D_Buffer(noise_aug_strength=0.25, generator=torch.Generator(device="cuda").manual_seed(3), **kw)
    p0, m0 = clean.render_cache(w2cs, Ks)
    p1, m1 = noisy.render_cache(w2cs, Ks)
    assert torch.equal(m0, m1)
    d = p1 - p0
    assert float(d[:, :, 1].abs().max()) < 1e-5   # two renders differ by the order of their float atomics only
    assert abs(float(d[:, :, 0].std()) - 0.25) < 0.01


@pytest.mark.parametrize("method", ["rigid", "non_rigid"])
def test_update_cache_with_depth_alignment_matches_reference(g, method):
    """update_cache's DEFAULT path: render the cache depth at the new pose, align the incoming depth to it (affine
    inverse-depth fit, then 100 Adam steps on a per-pixel scale map = g3c_align_depth_nonrigid), unproject, insert
    (reference cache_3d.py:262-316, camera_utils.py:225-347)."""
    c3, K, w2cs, Ks = _targets()
    cache = _buffer(c3, K)
    cache.update_cache(cu(c3["image"][1:2]), cu(g["align_new_depth"]), cu(g["buf_new_w2c"]), new_intrinsics=K,
                       depth_alignment=True, alignment_method=method)
    pts = cache.input_points[:, :, 0, 0].cpu().numpy()
    ref = g[f"align_{method}_points"]
    tm = g["align_target_mask"][0, 0, 0] > 0
    err = np.abs(pts - ref).max(-1)[0, 0] / np.abs(ref).max(-1)[0, 0].clip(1e-3)
    print(f"{method}: point error rel. to |p|: in-mask max {err[tm].max():.2e} mean {err[tm].mean():.2e}; "
          f"outside max {err[~tm].max():.2e}")
    # the target depth / mask come from this repo's render (a few coverage flips against the reference's): quantiles
    q_in, q_out = np.quantile(err[tm], 0.995), np.quantile(err[~tm], 0.99)
    assert q_in < (2e-4 if method == "rigid" else 3e-3) and err[tm].mean() < (5e-5 if method == "rigid" else 5e-4)
    assert q_out < (2e-4 if method == "rigid" else 1e-2)
    same_render(*cache.render_cache(w2cs, Ks), g[f"align_{method}_pixels"], g[f"align_{method}_masks"], atol=2e-2,
                flips=1e-2, frac=0.99)
    with pytest.raises(NotImplementedError):
        cache.update_cache(cu(c3["image"][1:2]), cu(g["align_new_depth"]), cu(g["buf_new_w2c"]), new_intrinsics=K,
                           alignment_method="affine")


def test_align_depth_native_matches_reference(g):
    from gen3c_b200 import camera_utils

    nd, td = cu(g["align_new_depth"][0, 0]), cu(g["align_target_depth"][0, 0])
    tmn = g["align_target_mask"][0, 0, 0] > 0
    tm = cu(tmn)
    K = cu(cases.warp_case("R3")["K"][0])
    c2w = torch.inverse(cu(g["buf_new_w2c"][0]))
    rigid = camera_utils.align_depth(nd, td, tm).cpu().numpy()
    np.testing.assert_allclose(rigid, g["align_rigid_depth"], rtol=5e-5)
    non = camera_utils.align_depth(nd, td, tm, k=K, c2w=c2w, alignment_method="non_rigid").cpu().numpy()
    ref = g["align_nonrigid_depth"]
    rel = np.abs(non - ref) / ref
    print(f"non-rigid: in-mask max {rel[tmn].max():.2e} mean {rel[tmn].mean():.2e}; outside max {rel[~tmn].max():.2e}")
    assert rel[tmn].max() < 2e-3 and rel[tmn].mean() < 4e-4 and rel[~tmn].max() < 8e-3
    assert (np.abs(non - rigid) / ref).mean() > 5e-3   # negative control: the second stage does something
    with pytest.raises(ValueError):
        camera_utils.align_depth(nd, td, tm, alignment_method="non_rigid")


def test_buffer_selector_and_cache4d_match_reference(g):
    from gen3c_b200.cache_3d import Cache3D_BufferSelector, Cache4D

    c3, K, w2cs, Ks = _targets()
    K3 = K[None].expand(1, 3, 3, 3).contiguous()
    sel = Cache3D_BufferSelector(frame_buffer_max=2, input_image=cu(g["sel_images"]), input_depth=cu(g["sel_depths"]),
                                 input_w2c=cu(g["sel_w2c"]), input_intrinsics=K3, input_format=["B", "N", "C", "H", "W"],
                                 filter_points_threshold=0.05)
    ps, ms = sel.render_cache(w2cs, Ks)
    assert ps.shape == (1, 2, 2, 3, 96, 128)
    same_render(ps, ms, g["sel_pixels"], g["sel_masks"])
    with pytest.raises(NotImplementedError):
        sel.update_cache()
    c4 = Cache4D(input_image=cu(g["sel_images"]), input_depth=cu(g["sel_depths"]), input_w2c=cu(g["sel_w2c"]),
                 input_intrinsics=K3, input_format=["B", "F", "C", "H", "W"], filter_points_threshold=0.05)
    assert c4.input_frame_count() == 3
    same_render(*c4.render_cache(w2cs, Ks, start_frame_idx=1), g["c4_pixels"], g["c4_masks"])
    with pytest.raises(RuntimeError):
        c4.render_cache(w2cs, Ks, start_frame_idx=2)   # only one cache frame left for two targets


def test_unproject_ray_depth_and_forward_warp_from_depth(g):
    """unproject_points(is_depth=False) (depth = distance along the ray, reference :445-448) and forward_warp with
    depth1 / transformation1 given instead of world points (:226-243, compute_transformed_points :523-573)."""
    from gen3c_b200 import warp

    c6 = cases.warp_case("R6")
    pr = warp.unproject_points(cu(c6["depth"]), cu(c6["w2c_src"]), cu(c6["K"]), is_depth=False)
    np.testing.assert_allclose(pr.cpu().numpy(), g["ray_points"], atol=5e-5, rtol=1e-5)
    for is_depth, tag in ((True, "d1"), (False, "d1r")):
        w, m, d, f = warp.forward_warp(cu(c6["image"]), None, cu(c6["depth"]), cu(c6["w2c_src"]), cu(c6["w2c_tgt"]),
                                       cu(c6["K"]), None, render_depth=is_depth, is_depth=is_depth)
        np.testing.assert_allclose(f.cpu().numpy(), g[f"{tag}_flow"], atol=3e-3)
        same_render(w, m, g[f"{tag}_warped"], g[f"{tag}_mask"])
        if is_depth:
            ok = (m.cpu().numpy() == g["d1_mask"])[:, 0] & (g["d1_mask"][:, 0] > 0)
            assert (np.abs(d.cpu().numpy()[ok] - g["d1_depth"][ok]) <= 1e-3).mean() > 0.999
