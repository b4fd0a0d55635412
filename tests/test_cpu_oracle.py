"""CPU suite: the restated oracles against the golden vectors minted from the reference's own code
(oracle/make_golden.py), host-side logic, and the C-ABI library's exported surface."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import cases, dit_oracle, golden, warp_oracle


@pytest.mark.parametrize("name", ["R1", "R2", "R3", "R4", "R5", "R6"])
def test_warp_oracle_matches_reference_golden(name, golden_dir):
    g = golden.load(golden_dir, f"warp_{name}")
    c = cases.warp_case(name)
    pts = warp_oracle.unproject_points(c["depth"], c["w2c_src"], c["K"])
    np.testing.assert_allclose(pts, g["points"], atol=2e-5, rtol=1e-5)
    w, m, d, f = warp_oracle.forward_warp(c["image"], c["mask"], g["points"], c["w2c_tgt"], c["K"], render_depth=True)
    np.testing.assert_allclose(f, g["flow"], atol=1e-4)
    assert np.array_equal(m, g["mask"])
    np.testing.assert_allclose(w, g["warped"], atol=1e-4)
    np.testing.assert_allclose(d, g["depth"], atol=1e-5)
    # the integer part is bit-exact on identical coordinates
    _, fl, ce = warp_oracle.splat_indices(g["flow"])
    assert np.array_equal(fl.astype(np.int32), g["floor"])
    assert np.array_equal(ce.astype(np.int32), g["ceil"])


def test_foreground_masking_oracle_matches_reference_golden(golden_dir):
    """SURVEY.md §8f rank 1 (next row): forward_warp(foreground_masking=True).  The golden comes from the reference's own
    forward_warp / points_to_mesh / get_camera_rays run on CPU; only the NVIDIA-Warp ray/triangle kernel is replaced by
    a torch restatement there (oracle/make_golden.py::torch_ray_triangle)."""
    g = golden.load(golden_dir, "warp_R7_foreground")
    c = cases.foreground_case()
    boundary = ~warp_oracle.reliable_depth_mask_range_batch(c["depth"]).astype(bool)[:, 0]
    assert np.array_equal(boundary, g["boundary"])
    w, m, d, _ = warp_oracle.forward_warp(c["image"], None, g["points"], c["w2c_tgt"], c["K"], foreground_masking=True,
                                          boundary_mask=boundary)
    assert np.array_equal(m, g["mask"])
    np.testing.assert_allclose(w, g["warped"], atol=1e-4)
    np.testing.assert_allclose(d, g["depth"], atol=1e-5)
    occluded = (g["mask_plain"] > 0) & (g["mask"] == 0)
    assert 0.02 < occluded.mean() < 0.06  # the near box hides a strip of background behind its edge
    assert np.all(w[0][:, occluded[0, 0]] == -1.0)  # killed pixels carry the fill value of an image


def test_ray_triangle_known_answers():
    """Moeller-Trumbore restatement on hand-checkable geometry: a unit right triangle at z = 2."""
    v = np.array([[0, 0, 2], [1, 0, 2], [0, 1, 2]], dtype=np.float32)
    f = np.array([[0, 1, 2]])
    d = np.array([[0.1, 0.1, 1.0], [0.6, 0.6, 1.0], [0.0, 0.0, -1.0], [0.25, 0.25, 1.0]], dtype=np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    t = warp_oracle.ray_triangle_depth(np.zeros_like(d), d, v, f)
    np.testing.assert_allclose(t[0] * d[0, 2], 2.0, rtol=1e-6)   # inside: z-depth of the plane
    assert t[1] == 0.0 and t[2] == 0.0                           # u + v > 1 ; behind the camera
    np.testing.assert_allclose(t[3] * d[3, 2], 2.0, rtol=1e-6)
    # nearest of two parallel triangles wins
    v2 = np.concatenate([v, v + np.array([0, 0, 1], dtype=np.float32)])
    t2 = warp_oracle.ray_triangle_depth(np.zeros_like(d), d, v2, np.array([[3, 4, 5], [0, 1, 2]]))
    np.testing.assert_allclose(t2[0] * d[0, 2], 2.0, rtol=1e-6)


def test_identity_camera_kat():
    """SURVEY.md §8d config 1: 256x256, identity camera, smooth depth -> image reproduced, mask all ones."""
    c = cases.warp_case("R1")
    pts = warp_oracle.unproject_points(c["depth"], c["w2c_src"], c["K"])
    w, m, _, _ = warp_oracle.forward_warp(c["image"], None, pts, c["w2c_tgt"], c["K"])
    assert m.min() == 1.0
    assert np.abs(w - c["image"]).max() <= 5e-4


def test_integer_coordinates_degenerate_kat():
    """KAT-R5: integer target coordinates -> floor == ceil, four unit weights on one pixel."""
    flow = np.full((1, 2, 8, 8), 2.0, dtype=np.float32)
    _, fl, ce = warp_oracle.splat_indices(flow)
    assert np.array_equal(fl, ce)
    img = np.random.RandomState(0).uniform(-1, 1, (1, 3, 8, 8)).astype(np.float32)
    out, mask = warp_oracle.bilinear_splatting(img, None, np.ones((1, 1, 8, 8), np.float32), flow, is_image=True)
    np.testing.assert_allclose(out[:, :, 2:, 2:], img[:, :, :-2, :-2], atol=1e-6)
    assert mask[:, :, :2].max() == 0 and mask[:, :, :, :2].max() == 0


def test_chunk_coupling_kat():
    """KAT-R3: the log-depth max is shared by the items of one call; normalised outputs still agree."""
    c = cases.warp_case("R3")
    pts = warp_oracle.unproject_points(c["depth"], c["w2c_src"], c["K"])
    both = warp_oracle.forward_warp(c["image"], None, pts, c["w2c_tgt"], c["K"])[0]
    solo = warp_oracle.forward_warp(c["image"][:1], None, pts[:1], c["w2c_tgt"][:1], c["K"][:1])[0]
    assert np.abs(both[:1] - solo).max() < 5e-2  # different soft-z sharpness, same picture


def test_render_cache_oracle_matches_reference(golden_dir):
    g = golden.load(golden_dir, "warp_cache")
    c = cases.warp_case("R3")
    F = 3
    w2cs = cases.pan_trajectory(F, 0.1)[None]
    Ks = np.tile(c["K"][:1], (F, 1, 1))[None]
    img = c["image"][None, None]  # (B=1, Fs=1, N=2, 3, H, W)
    pix, msk = warp_oracle.render_cache(g["points"], img, g["cache_mask"], w2cs, Ks)
    # the oracle re-projects with numpy's matmul (rounding order differs from torch's): sub-pixel positions
    # move by ~1e-5 px, which the soft-z weights amplify
    assert (msk != g["masks"]).mean() < 1e-3
    assert np.abs(pix - g["pixels"]).mean() < 1e-5 and (np.abs(pix - g["pixels"]) <= 2e-3).mean() > 0.999
    rel = warp_oracle.reliable_depth_mask_range_batch(c["depth"].reshape(-1, 1, 96, 128), ratio_thresh=0.05)
    assert np.array_equal(rel, g["reliable"])


def test_dit_oracle_matches_reference_golden(golden_dir):
    g = golden.load(golden_dir, "dit_tiny")
    cfg, shp = cases.TINY, cases.TINY_SHAPE
    sd = dit_oracle.random_state_dict(cfg, seed=0)
    inp = cases.dit_inputs(cfg, **shp)
    oc = dit_oracle.forward(sd, cfg, inp["x"], inp["cond_mask"], inp["pose"], inp["padding"], inp["timestep"], inp["ctx_c"])
    ou = dit_oracle.forward(sd, cfg, inp["x"], inp["cond_mask"], None, inp["padding"], inp["timestep"], inp["ctx_u"])
    for o, ref in ((oc, g["out_cond"]), (ou, g["out_uncond"])):
        ref = torch.from_numpy(ref)
        assert float((o - ref).norm() / ref.norm()) < 1e-5


def test_scheduler_host_logic():
    from gen3c_b200.sampler import EDMEulerScheduler

    s = EDMEulerScheduler().set_timesteps(35)
    ref = dit_oracle.karras_sigmas(35)
    np.testing.assert_allclose(s.sigmas, ref, rtol=1e-6)
    assert abs(s.sigmas[0] - 80.0) < 1e-4 and abs(s.sigmas[34] - 0.0002) < 1e-7 and s.sigmas[35] == 0
    assert abs(s.init_noise_sigma - (80 ** 2 + 1) ** 0.5) < 1e-9
    np.testing.assert_allclose(s.timesteps, 0.25 * np.log(ref[:-1]), rtol=1e-6)


def test_c_abi_exports_every_declared_symbol():
    """The shared library loads without a GPU and exports exactly what include/gen3c_b200.h declares."""
    from gen3c_b200 import _lib

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, "include", "gen3c_b200.h")).read()
    declared = set(re.findall(r"\b(g3c_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.g3c_version() >= 100
    assert isinstance(lib.g3c_last_error(), bytes)


def test_product_path_never_imports_oracle():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for dirpath, _, files in os.walk(os.path.join(root, "gen3c_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("# oracle-free", ""), f"{f} mentions the oracle"


def test_condition_assembly_host_logic():
    """D12: add_condition_video_indicator_and_video_input_mask / encode_warped_frames / add_condition_pose against the
    reference semantics (model_v2w.py:32-82, model_gen3c.py:32-57,115-139) with a synthetic encoder."""
    from gen3c_b200 import model_gen3c as mg

    B, T, H, W = 1, 4, 8, 8
    lat = torch.randn(B, 16, T, H, W)
    c = mg.VideoExtendCondition(crossattn_emb=torch.zeros(1, 4, 8), video_cond_bool=True)
    c = mg.add_condition_video_indicator_and_video_input_mask(lat, c, num_condition_t=1)
    assert c.condition_video_indicator.shape == (1, 1, T, 1, 1) and float(c.condition_video_indicator.sum()) == 1.0
    assert c.condition_video_input_mask.shape == (B, 1, T, H, W)
    assert float(c.condition_video_input_mask[:, :, 0].min()) == 1.0 and float(c.condition_video_input_mask[:, :, 1:].max()) == 0.0
    u = mg.VideoExtendCondition(crossattn_emb=torch.zeros(1, 4, 8), video_cond_bool=False)
    u = mg.add_condition_video_indicator_and_video_input_mask(lat, u, 1)
    assert float(u.condition_video_input_mask.abs().max()) == 0.0
    with pytest.raises(AssertionError):
        mg.add_condition_video_indicator_and_video_input_mask(lat, c, None)

    F = 9
    enc_calls = []

    def encode(x):  # [B,3,F,h,w] -> [B,16,T,H,W]
        enc_calls.append(float(x.float().mean()))
        return torch.full((B, 16, T, H, W), float(x.float().mean()))

    state = torch.rand(B, F, 1, 3, 16, 16)           # one buffer, frame_buffer_max = 2 -> zero padded
    mask = torch.ones(B, F, 1, 1, 16, 16)
    lc = mg.encode_warped_frames(state, mask, encode, frame_buffer_max=2, dtype=torch.float32)
    assert lc.shape == (B, 64, T, H, W)
    assert abs(enc_calls[1] - 1.0) < 1e-6            # mask * 2 - 1 = 1, repeated to 3 channels
    assert float(lc[:, 32:].abs().max()) == 0.0      # second buffer slot is zero
    c = mg.add_condition_pose(lc, c)
    u = mg.add_condition_pose(lc, u, drop_out_latent=True)
    assert torch.equal(c.condition_video_pose, lc) and float(u.condition_video_pose.abs().max()) == 0.0
    cond, uncond = mg.get_conditions(torch.zeros(1, 4, 8), torch.ones(1, 4, 8), torch.zeros(1, 1, 16, 16), state, mask, lat,
                                     1, encode, dtype=torch.float32)
    assert torch.equal(cond.condition_video_input_mask, uncond.condition_video_input_mask)  # add_input_frames_guidance=False
    assert set(cond.to_dict()) >= {"crossattn_emb", "condition_video_pose", "condition_video_input_mask", "gt_latent"}
