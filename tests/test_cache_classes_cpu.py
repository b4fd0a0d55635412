"""CPU checks of the host logic either side of Path R against goldens minted from the reference's own code
(tests/golden/warp_cache_classes.npz, oracle/make_golden.py::mint_cache_classes): camera trajectories, the rigid
inverse-depth fit, and the restated (closed-form gradient) non-rigid depth alignment of the oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import cases, golden, warp_oracle


@pytest.fixture(scope="module")
def g(golden_dir):
    return golden.load(golden_dir, "warp_cache_classes")


def test_camera_trajectories_match_reference(g):
    from gen3c_b200 import camera_utils as cu

    w0 = torch.from_numpy(g["traj_w0"])
    K = torch.from_numpy(cases.warp_case("R3")["K"][0])
    for ty in ("left", "right", "up", "down", "zoom_in", "zoom_out", "clockwise", "counterclockwise"):
        for rot in ("center_facing", "no_rotation", "trajectory_aligned"):
            w2, k2 = cu.generate_camera_trajectory(ty, w0, K, 7, 0.3, rot, center_depth=1.7, device="cpu")
            assert k2.shape == (1, 7, 3, 3)
            np.testing.assert_allclose(w2.numpy(), g[f"traj_{ty}_{rot}"], atol=1e-6, rtol=1e-6)
    with pytest.raises(ValueError):
        cu.generate_camera_trajectory("sideways", w0, K, 7, 0.3, "center_facing", device="cpu")
    with pytest.raises(ValueError):
        cu.generate_camera_trajectory("left", w0, K, 7, 0.3, "upside_down", device="cpu")


def _alignment_inputs(g):
    nd = g["align_new_depth"][0, 0]
    td = g["align_target_depth"][0, 0]
    tm = g["align_target_mask"][0, 0, 0] > 0
    K = cases.warp_case("R3")["K"][0]
    c2w = np.linalg.inv(g["buf_new_w2c"][0]).astype(np.float32)
    return nd, td, tm, K, c2w


def test_rigid_alignment_host_mirror_and_oracle_match_reference(g):
    from gen3c_b200 import camera_utils as cu

    nd, td, tm, _, _ = _alignment_inputs(g)
    ref = g["align_rigid_depth"]
    np.testing.assert_allclose(warp_oracle.align_depth(nd, td, tm), ref, rtol=2e-6)
    got = cu._align_inv_depth_to_depth(1.0 / torch.from_numpy(nd), torch.from_numpy(td), torch.from_numpy(tm)).numpy()
    np.testing.assert_allclose(got, ref, rtol=2e-5)


def test_nonrigid_alignment_oracle_matches_reference_autograd(g):
    """The oracle writes the gradient of the reference's loss out by hand; the reference differentiates with autograd and
    steps torch.optim.Adam.  100 iterations of sign-gradient dynamics agree to < 1e-3 of the depth inside the target mask
    (measured 8.6e-4 max, 1.5e-4 mean) and to 3e-3 outside it, where only the smoothness term acts."""
    nd, td, tm, K, c2w = _alignment_inputs(g)
    got = warp_oracle.align_depth(nd, td, tm, k=K, c2w=c2w, alignment_method="non_rigid")
    ref = g["align_nonrigid_depth"]
    rel = np.abs(got - ref) / ref
    assert rel[tm].max() < 1.5e-3 and rel[tm].mean() < 3e-4
    assert rel[~tm].max() < 5e-3
    # and it is not the rigid result: the non-rigid stage moves the depth by ~1e-2
    assert (np.abs(ref - g["align_rigid_depth"]) / ref).mean() > 5e-3
