"""Mint the golden vectors under tests/golden/ by executing the REFERENCE'S OWN code (imported from
/root/reference through oracle/ref_stubs.py) on the seeded cases of oracle/cases.py, and check the
restated oracles (oracle/warp_oracle.py, oracle/dit_oracle.py) against it while doing so.

Run in the build container only:   python -m oracle.make_golden
The reference ships no golden vectors for either hot path (SURVEY.md §4); these fixtures are the pins.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

from . import cases, dit_oracle, golden, ref_stubs, warp_oracle

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def mint_warp():
    ref = ref_stubs.reference_warp_module()
    report = []
    for name in ("R1", "R2", "R3", "R4", "R5", "R6"):
        c = cases.warp_case(name)
        with torch.no_grad():
            pts = ref.unproject_points(t(c["depth"]), t(c["w2c_src"]), t(c["K"]), is_depth=True)
            warped, mask, depth, flow = ref.forward_warp(
                t(c["image"]), None if c["mask"] is None else t(c["mask"]), None, None, t(c["w2c_tgt"]),
                t(c["K"]), t(c["K"]), render_depth=True, world_points1=pts)
        pts_o = warp_oracle.unproject_points(c["depth"], c["w2c_src"], c["K"])
        # feed the oracle the reference's points so that the splat is compared on identical inputs
        w_o, m_o, d_o, f_o = warp_oracle.forward_warp(c["image"], c["mask"], pts.numpy(), c["w2c_tgt"], c["K"],
                                                      render_depth=True)
        e_pts = float(np.abs(pts_o - pts.numpy()).max())
        e_img = float(np.abs(w_o - warped.numpy()).max())
        e_msk = float(np.abs(m_o - mask.numpy()).max())
        e_dep = float(np.abs(d_o - depth.numpy()).max())
        e_flow = float(np.abs(f_o - flow.numpy()).max())
        # integer indices on the reference's own flow: must be bit-exact
        _, fl, ce = warp_oracle.splat_indices(flow.numpy())
        b, _, h, w = flow.shape
        grid = ref.create_grid(b, h, w)
        pos = flow + grid + 1
        rfl = torch.floor(pos).long()
        rce = torch.ceil(pos).long()
        lim = torch.tensor([w + 1, h + 1]).view(1, 2, 1, 1)
        rfl = torch.minimum(torch.clamp(rfl, min=0), lim)
        rce = torch.minimum(torch.clamp(rce, min=0), lim)
        idx_equal = bool((t(fl) == rfl).all() and (t(ce) == rce).all())
        report.append((name, e_pts, e_img, e_msk, e_dep, e_flow, idx_equal, float(mask.mean())))
        golden.save(OUT, f"warp_{name}", points=pts.numpy(), warped=warped.numpy(),
                            mask=mask.numpy(), depth=depth.numpy(), flow=flow.numpy(),
                            floor=rfl.numpy().astype(np.int32), ceil=rce.numpy().astype(np.int32))
    # reliability mask + render_cache chunking through the reference's Cache3D_Buffer (N = 2 buffers)
    cache_mod = ref_stubs.reference_cache_module()
    c = cases.warp_case("R3")
    F = 3
    w2cs = t(cases.pan_trajectory(F, 0.1))[None]
    Ks = t(np.tile(c["K"][:1], (F, 1, 1)))[None]
    cache = cache_mod.Cache3D_Buffer(
        frame_buffer_max=2, noise_aug_strength=0, generator=None,
        input_image=t(c["image"])[None], input_depth=t(c["depth"])[None], input_w2c=t(c["w2c_src"])[None],
        input_intrinsics=t(c["K"])[None], input_format=["B", "N", "C", "H", "W"], device="cpu",
        filter_points_threshold=0.05, foreground_masking=False)
    with torch.no_grad():
        pix, msk = cache_mod.Cache3D_Base.render_cache(cache, w2cs, Ks)
    rel = ref.reliable_depth_mask_range_batch(t(c["depth"]).reshape(-1, 1, 96, 128), ratio_thresh=0.05)
    rel_o = warp_oracle.reliable_depth_mask_range_batch(c["depth"].reshape(-1, 1, 96, 128), ratio_thresh=0.05)
    pts2 = cache.input_points.numpy()[:, :, :, 0]
    img2 = cache.input_image.numpy()[:, :, :, 0]
    m2 = cache.input_mask.numpy()[:, :, :, 0].astype(np.float32)
    pix_o, msk_o = warp_oracle.render_cache(pts2, img2, m2, w2cs.numpy(), Ks.numpy())
    e_cache = float(np.abs(pix_o - pix.numpy()).max())
    golden.save(OUT, "warp_cache", pixels=pix.numpy(), masks=msk.numpy(),
                        reliable=rel.numpy(), points=pts2, cache_mask=m2)
    print("== Path R: restated oracle vs reference (max abs err) ==")
    for r in report:
        print("  %s  points %.2e  image %.2e  mask %.1f  depth %.2e  flow %.2e  indices_bit_exact=%s  coverage %.3f" % r)
    print("  render_cache(N=2, F=3, chunk 2): image %.2e ; reliable-mask equal: %s" %
          (e_cache, bool((rel.numpy() == rel_o).all())))
    bad = [r for r in report if r[2] > 2e-3 or not r[6] or r[3] > 0]
    if bad or e_cache > 2e-3:
        print("!! restated warp oracle disagrees with the reference:", bad, e_cache)
        return 1
    return mint_foreground(ref)


def torch_ray_triangle(ray_origins, ray_directions, vertices, faces, device):
    """Stand-in for the NVIDIA Warp kernel (ray_triangle_intersection_warp.py:23-105, launched at :243-258 / :267-287),
    which needs Warp + CUDA: the same Moeller-Trumbore test, brute force in float32 torch.  Everything else on the
    foreground-masking path below is the reference's own code."""
    H, W = ray_origins.shape[:2]
    o, d = ray_origins.reshape(-1, 1, 3).float(), ray_directions.reshape(-1, 1, 3).float()
    v0, v1, v2 = vertices[faces[:, 0]][None], vertices[faces[:, 1]][None], vertices[faces[:, 2]][None]
    e1, e2 = v1 - v0, v2 - v0
    h = torch.cross(d.expand(-1, e2.shape[1], -1), e2.expand(d.shape[0], -1, -1), dim=-1)
    a = (e1 * h).sum(-1)
    ok = a.abs() >= 1e-8
    f = 1.0 / a
    s = o - v0
    u = f * (s * h).sum(-1)
    ok &= ~((u < 0) | (u > 1))
    q = torch.cross(s, e1.expand(s.shape[0], -1, -1), dim=-1)
    v = f * (d * q).sum(-1)
    ok &= ~((v < 0) | (u + v > 1))
    tt = f * (e2 * q).sum(-1)
    ok &= tt > 1e-8
    tt = torch.where(ok, tt, torch.full_like(tt, 1e10))
    best = tt.min(dim=1).values
    return torch.where(best < 1e10, best, torch.zeros_like(best)).reshape(H, W)


def mint_foreground(ref):
    """forward_warp(foreground_masking=True) of the reference on CPU (R7) -> tests/golden/warp_R7_foreground.npz."""
    ref._warp_initialized = True
    ref._ray_triangle_intersection_func = torch_ray_triangle
    c = cases.foreground_case()
    with torch.no_grad():
        pts = ref.unproject_points(t(c["depth"]), t(c["w2c_src"]), t(c["K"]), is_depth=True)
        boundary = ~ref.reliable_depth_mask_range_batch(t(c["depth"]))[:, 0]
        base = ref.forward_warp(t(c["image"]), None, None, None, t(c["w2c_tgt"]), t(c["K"]), t(c["K"]), render_depth=True,
                                world_points1=pts)
        warped, mask, depth, flow = ref.forward_warp(t(c["image"]), None, None, None, t(c["w2c_tgt"]), t(c["K"]), t(c["K"]),
                                                     world_points1=pts, foreground_masking=True, boundary_mask=boundary)
    b_o = ~(warp_oracle.reliable_depth_mask_range_batch(c["depth"]).astype(bool)[:, 0])
    w_o, m_o, d_o, _ = warp_oracle.forward_warp(c["image"], None, pts.numpy(), c["w2c_tgt"], c["K"], foreground_masking=True,
                                                boundary_mask=b_o)
    killed = float(((base[1] > 0) & (mask == 0)).float().mean())
    flips = float((m_o != mask.numpy()).mean())
    same = (m_o == mask.numpy())[:, 0]
    e_img = float(np.abs(w_o - warped.numpy())[np.broadcast_to(same[:, None], w_o.shape)].max())
    print("Path R foreground masking (R7): boundary px %.3f, occluded px %.4f, oracle mask flips %.2e, image err %.2e, "
          "boundary mask equal: %s" % (float(boundary.float().mean()), killed, flips, e_img,
                                       bool((b_o == boundary.numpy()).all())))
    golden.save(OUT, "warp_R7_foreground", points=pts.numpy(), boundary=boundary.numpy(),
                        warped=warped.numpy(), mask=mask.numpy(), depth=depth.numpy(), mask_plain=base[1].numpy())
    return 0 if (killed > 0.005 and flips < 2e-3 and e_img < 2e-3) else 1


def mint_dit():
    Net = ref_stubs.reference_dit_class()
    from cosmos_predict1.diffusion.conditioner import DataType

    cfg, shp = cases.TINY, cases.TINY_SHAPE
    net = Net(max_img_h=cfg.max_h * 2, max_img_w=cfg.max_w * 2, max_frames=cfg.max_frames, in_channels=cfg.in_channels,
              out_channels=cfg.out_channels, patch_spatial=2, patch_temporal=1, model_channels=cfg.model_channels,
              block_config="FA-CA-MLP", num_blocks=cfg.num_blocks, num_heads=cfg.num_heads, concat_padding_mask=True,
              pos_emb_cls="rope3d", pos_emb_learnable=False, pos_emb_interpolation="crop", block_x_format="THWBD",
              affline_emb_norm=True, use_adaln_lora=True, adaln_lora_dim=cfg.adaln_lora_dim,
              rope_t_extrapolation_ratio=cfg.rope_t_ratio, crossattn_emb_channels=cfg.context_dim)
    sd = dit_oracle.random_state_dict(cfg, seed=0)
    missing, unexpected = net.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all("_extra_state" in m for m in missing), missing
    net.eval()
    inp = cases.dit_inputs(cfg, **shp)

    def run(net, dtype, pose, ctx):
        kw = dict(
            x=inp["x"][None].to(dtype), timesteps=torch.tensor([inp["timestep"]], dtype=dtype),
            crossattn_emb=ctx[None].to(dtype), crossattn_mask=None, fps=torch.tensor([24.0]),
            image_size=None, padding_mask=inp["padding"][None, None].to(dtype), data_type=DataType.VIDEO,
            condition_video_input_mask=inp["cond_mask"][None].to(dtype),
            condition_video_indicator=torch.zeros(1, 1, shp["T"], 1, 1, dtype=dtype),
            condition_video_pose=pose[None].to(dtype))
        with torch.no_grad():
            return net(**kw)[0].float()

    out_c = run(net, torch.float32, inp["pose"], inp["ctx_c"])
    out_u = run(net, torch.float32, torch.zeros_like(inp["pose"]), inp["ctx_u"])
    o_c = dit_oracle.forward(sd, cfg, inp["x"], inp["cond_mask"], inp["pose"], inp["padding"], inp["timestep"], inp["ctx_c"])
    o_u = dit_oracle.forward(sd, cfg, inp["x"], inp["cond_mask"], None, inp["padding"], inp["timestep"], inp["ctx_u"])

    def rel(a, b):
        return float((a - b).norm() / b.norm())

    e_c, e_u = rel(o_c, out_c), rel(o_u, out_u)
    # the reference's own bf16 noise floor (same graph, bf16 weights + activations) vs its fp32 run
    net_bf = Net(max_img_h=cfg.max_h * 2, max_img_w=cfg.max_w * 2, max_frames=cfg.max_frames, in_channels=cfg.in_channels,
                 out_channels=cfg.out_channels, patch_spatial=2, patch_temporal=1, model_channels=cfg.model_channels,
                 block_config="FA-CA-MLP", num_blocks=cfg.num_blocks, num_heads=cfg.num_heads, concat_padding_mask=True,
                 pos_emb_cls="rope3d", pos_emb_learnable=False, pos_emb_interpolation="crop", block_x_format="THWBD",
                 affline_emb_norm=True, use_adaln_lora=True, adaln_lora_dim=cfg.adaln_lora_dim,
                 rope_t_extrapolation_ratio=cfg.rope_t_ratio, crossattn_emb_channels=cfg.context_dim)
    net_bf.load_state_dict(sd, strict=False)
    net_bf = net_bf.to(torch.bfloat16).eval()
    out_c_bf = run(net_bf, torch.bfloat16, inp["pose"], inp["ctx_c"])
    floor = rel(out_c_bf, out_c)
    golden.save(OUT, "dit_tiny", out_cond=out_c.numpy(), out_uncond=out_u.numpy(),
                        ref_bf16_rel_l2=np.float32(floor))
    print("== Path D (tiny 2-block, D=256, L=128): restated oracle vs reference fp32 forward ==")
    print("  rel-L2 cond %.2e  uncond %.2e ; reference bf16-vs-fp32 noise floor rel-L2 %.2e" % (e_c, e_u, floor))
    if e_c > 1e-4 or e_u > 1e-4:
        print("!! restated DiT oracle disagrees with the reference")
        return 1
    return 0


def mint_cache_classes():
    """The reference's own Cache3D_Buffer / Cache3D_BufferSelector / Cache4D objects (cache_3d.py:26-433) and align_depth
    (camera_utils.py:225-347) executed on CPU -> tests/golden/warp_cache_classes.npz: ring of 2 with
    update_cache(depth_alignment=False), the rigid and non-rigid depth alignment of update_cache (default arguments),
    top-K buffer selection, per-frame 4D cache, unproject_points(is_depth=False) and forward_warp(depth1=...)."""
    ref = ref_stubs.reference_warp_module()
    cm = ref_stubs.reference_cache_module()
    import cosmos_predict1.diffusion.inference.camera_utils as cu

    out = {}
    c3, c6 = cases.warp_case("R3"), cases.warp_case("R6")
    h, w = 96, 128
    K = t(c3["K"][:1])
    F = 2
    w2cs = t(cases.pan_trajectory(F, 0.08))[None]
    Ks = K[None].expand(1, F, 3, 3).contiguous()
    # ---- Cache3D_Buffer: ring of 2, three inserts (append, then overwrite slot 0 twice), no alignment
    cache = cm.Cache3D_Buffer(frame_buffer_max=2, noise_aug_strength=0, generator=None,
                              input_image=t(c3["image"][:1]), input_depth=t(c3["depth"][:1]), input_w2c=t(c3["w2c_src"][:1]),
                              input_intrinsics=K, device="cpu", filter_points_threshold=0.05, foreground_masking=False)
    with torch.no_grad():
        p0, m0 = cache.render_cache(w2cs, Ks)
        new_w2c = t(cases.look(0.02, -0.01, (0.03, 0.0, 0.01)))[None]
        cache.update_cache(t(c3["image"][1:2]), t(c3["depth"][1:2]), new_w2c, new_intrinsics=K, depth_alignment=False)
        p1, m1 = cache.render_cache(w2cs, Ks)
        new_w2c2 = t(cases.look(-0.03, 0.005, (-0.02, 0.01, 0.0)))[None]
        cache.update_cache(t(c6["image"]), t(c6["depth"]), new_w2c2, new_intrinsics=K, depth_alignment=False)
        p2, m2 = cache.render_cache(w2cs, Ks)
        d2, dm2 = cache.render_cache(w2cs, Ks, render_depth=True)
    out.update(buf_p0=p0.numpy(), buf_m0=m0.numpy(), buf_p1=p1.numpy(), buf_m1=m1.numpy(), buf_p2=p2.numpy(),
               buf_m2=m2.numpy(), buf_d2=d2.numpy(), buf_new_w2c=new_w2c.numpy(), buf_new_w2c2=new_w2c2.numpy())
    # ---- update_cache with depth alignment (the default path): rigid and non-rigid (100 Adam steps)
    for method in ("rigid", "non_rigid"):
        cache = cm.Cache3D_Buffer(frame_buffer_max=2, noise_aug_strength=0, generator=None,
                                  input_image=t(c3["image"][:1]), input_depth=t(c3["depth"][:1]), input_w2c=t(c3["w2c_src"][:1]),
                                  input_intrinsics=K, device="cpu", filter_points_threshold=0.05, foreground_masking=False)
        # a new depth map that disagrees with the cache by an affine map of inverse depth plus a smooth non-rigid part
        nd = c3["depth"][:1] * (1.15 + 0.05 * cases.smooth_depth(h, w)[None, None] / 3.5) + 0.2
        cache.update_cache(t(c3["image"][1:2]), t(nd.astype(np.float32)), new_w2c, new_intrinsics=K, depth_alignment=True,
                           alignment_method=method)
        with torch.no_grad():
            pa, ma = cache.render_cache(w2cs, Ks)
        out[f"align_{method}_points"] = cache.input_points[:, :, 0, 0].numpy()
        out[f"align_{method}_pixels"] = pa.numpy()
        out[f"align_{method}_masks"] = ma.numpy()
    out["align_new_depth"] = nd.astype(np.float32)
    # the aligned depth itself, from align_depth called the way update_cache calls it
    cache = cm.Cache3D_Buffer(frame_buffer_max=2, noise_aug_strength=0, generator=None,
                              input_image=t(c3["image"][:1]), input_depth=t(c3["depth"][:1]), input_w2c=t(c3["w2c_src"][:1]),
                              input_intrinsics=K, device="cpu", filter_points_threshold=0.05, foreground_masking=False)
    with torch.no_grad():
        td, tm = cache.render_cache(new_w2c.unsqueeze(1), K.unsqueeze(1), render_depth=True)
    td, tm = td[:, :, 0], tm[:, :, 0]
    rigid = cu.align_depth(t(nd.astype(np.float32)).squeeze(), td.squeeze(), tm.bool().squeeze())
    with torch.enable_grad():
        nonrigid = cu.align_depth(t(nd.astype(np.float32)).squeeze(), td.squeeze(), tm.bool().squeeze(), k=K.squeeze(),
                                  c2w=torch.inverse(new_w2c.squeeze()), alignment_method="non_rigid", num_iters=100,
                                  lambda_arap=0.1, smoothing_kernel_size=3).detach()
    out.update(align_target_depth=td.numpy(), align_target_mask=tm.numpy(), align_rigid_depth=rigid.numpy(),
               align_nonrigid_depth=nonrigid.numpy())
    # ---- Cache3D_BufferSelector: 3 buffers at init, keep the 2 with the largest overlap, near-full masking
    imgs = np.stack([c3["image"][0], c3["image"][1], c6["image"][0]])[None]          # B N C H W
    deps = np.stack([c3["depth"][0], c3["depth"][1], c6["depth"][0]])[None]
    srcs = np.stack([np.eye(4, dtype=np.float32), cases.look(0.3, 0.0, (0.6, 0.0, 0.0)), cases.look(-0.02, 0.0, (0.01, 0, 0))])[None]
    sel = cm.Cache3D_BufferSelector(frame_buffer_max=2, input_image=t(imgs), input_depth=t(deps), input_w2c=t(srcs),
                                    input_intrinsics=K[None].expand(1, 3, 3, 3).contiguous(),
                                    input_format=["B", "N", "C", "H", "W"], device="cpu", filter_points_threshold=0.05)
    with torch.no_grad():
        ps, ms = sel.render_cache(w2cs, Ks)
    out.update(sel_images=imgs, sel_depths=deps, sel_w2c=srcs, sel_pixels=ps.numpy(), sel_masks=ms.numpy())
    # ---- Cache4D: one cache frame per target frame, start_frame_idx = 1
    imgs4 = np.stack([c3["image"][0], c3["image"][1], c6["image"][0]])[None]         # B F C H W
    c4 = cm.Cache4D(input_image=t(imgs4), input_depth=t(deps), input_w2c=t(srcs),
                    input_intrinsics=K[None].expand(1, 3, 3, 3).contiguous(), input_format=["B", "F", "C", "H", "W"],
                    device="cpu", filter_points_threshold=0.05)
    with torch.no_grad():
        p4, m4 = c4.render_cache(w2cs, Ks, start_frame_idx=1)
    out.update(c4_pixels=p4.numpy(), c4_masks=m4.numpy())
    # ---- unproject_points(is_depth=False) and forward_warp with depth1 given (is_depth True / False)
    with torch.no_grad():
        pr = ref.unproject_points(t(c6["depth"]), t(c6["w2c_src"]), t(c6["K"]), is_depth=False)
        fw = ref.forward_warp(t(c6["image"]), None, t(c6["depth"]), t(c6["w2c_src"]), t(c6["w2c_tgt"]), t(c6["K"]), None,
                              render_depth=True)
        fr = ref.forward_warp(t(c6["image"]), None, t(c6["depth"]), t(c6["w2c_src"]), t(c6["w2c_tgt"]), t(c6["K"]), None,
                              is_depth=False)
    out.update(ray_points=pr.numpy(), d1_warped=fw[0].numpy(), d1_mask=fw[1].numpy(), d1_depth=fw[2].numpy(),
               d1_flow=fw[3].numpy(), d1r_warped=fr[0].numpy(), d1r_mask=fr[1].numpy(), d1r_flow=fr[3].numpy())
    # ---- camera trajectories (camera_utils.py:142-222), 4x4 host arithmetic
    w0 = t(cases.look(0.05, -0.02, (0.1, 0.0, 0.2)))
    for ty in ("left", "right", "up", "down", "zoom_in", "zoom_out", "clockwise", "counterclockwise"):
        for rot in ("center_facing", "no_rotation", "trajectory_aligned"):
            w2, k2 = cu.generate_camera_trajectory(ty, w0, K[0], 7, 0.3, rot, center_depth=1.7, device="cpu")
            out[f"traj_{ty}_{rot}"] = w2.numpy()
    out["traj_w0"] = w0.numpy()
    golden.save(OUT, "warp_cache_classes", **out)
    # the restated oracle against the same runs
    po = warp_oracle.unproject_points(c6["depth"], c6["w2c_src"], c6["K"], is_depth=False)
    print("== Path R classes: ring/selector/4D/alignment goldens written; oracle unproject(is_depth=False) err %.2e; "
          "non-rigid vs rigid depth change mean %.3e ==" % (float(np.abs(po - pr.numpy()).max()),
                                                              float((nonrigid - rigid).abs().mean())))
    return 0


def _ref_net(Net, cfg, **over):
    kw = dict(max_img_h=cfg.max_h * 2, max_img_w=cfg.max_w * 2, max_frames=cfg.max_frames, in_channels=cfg.in_channels,
              out_channels=cfg.out_channels, patch_spatial=2, patch_temporal=1, model_channels=cfg.model_channels,
              block_config="FA-CA-MLP", num_blocks=cfg.num_blocks, num_heads=cfg.num_heads, concat_padding_mask=True,
              pos_emb_cls="rope3d", pos_emb_learnable=False, pos_emb_interpolation="crop", block_x_format="THWBD",
              affline_emb_norm=True, use_adaln_lora=True, adaln_lora_dim=cfg.adaln_lora_dim,
              rope_t_extrapolation_ratio=cfg.rope_t_ratio, crossattn_emb_channels=cfg.context_dim)
    kw.update(over)
    return Net(**kw)


def mint_dit_fullwidth():
    """ONE block of the network at the full BASELINE width (D=4096, 32 heads, ffn 16 384, ctx 512x1024, position tables
    240/128) on two latent frames of the 720p grid (7 040 tokens), executed by the reference's own class in fp32 on the
    CPU -> tests/golden/dit_fullwidth.npz (output only: the weights are regenerated from the seed)."""
    Net = ref_stubs.reference_dit_class()
    from cosmos_predict1.diffusion.conditioner import DataType

    cfg, shp = cases.FULLWIDTH_1BLOCK, cases.FULLWIDTH_SHAPE
    sd = dit_oracle.random_state_dict(cfg, seed=21)
    net = _ref_net(Net, cfg)
    missing, unexpected = net.load_state_dict(sd, strict=False)
    assert not unexpected and all("_extra_state" in m for m in missing)
    net.eval()
    inp = cases.dit_inputs(cfg, **shp, seed=22)
    T = shp["T"]
    with torch.no_grad():
        out = net(x=inp["x"][None], timesteps=torch.tensor([inp["timestep"]]), crossattn_emb=inp["ctx_c"][None],
                  crossattn_mask=None, fps=torch.tensor([24.0]), image_size=None, padding_mask=inp["padding"][None, None],
                  data_type=DataType.VIDEO, condition_video_input_mask=inp["cond_mask"][None],
                  condition_video_indicator=torch.zeros(1, 1, T, 1, 1), condition_video_pose=inp["pose"][None])[0].float()
    o = dit_oracle.forward(sd, cfg, inp["x"], inp["cond_mask"], inp["pose"], inp["padding"], inp["timestep"], inp["ctx_c"])
    e = float((o - out).norm() / out.norm())
    ob = dit_oracle.forward({k: v.to(torch.bfloat16) for k, v in sd.items()}, cfg, inp["x"], inp["cond_mask"], inp["pose"],
                            inp["padding"], inp["timestep"], inp["ctx_c"], compute_dtype=torch.bfloat16).float()
    eb = float((ob - out).norm() / out.norm())
    golden.save(OUT, "dit_fullwidth", out_cond=out.numpy(), oracle_bf16_rel_l2=np.float32(eb))
    print("== Path D (1 block at full width D=4096/32 heads/ffn 16384/ctx 512x1024, 7 040 tokens): restated oracle vs the "
          "reference's fp32 forward rel-L2 %.2e ; bf16 run of the oracle vs it %.2e ==" % (e, eb))
    return 0 if e < 1e-4 else 1


def mint_tokenizer():
    """The reference's VideoJITTokenizer (module/pretrained_vae.py:314-509) on a tiny TorchScript checkpoint
    (oracle/cases.py::write_tiny_tokenizer) -> tests/golden/vae_wrapper.npz: chunked encode / decode, latent mean / std,
    dtype handling (fp32 and bf16 modules), frame-count helpers."""
    import tempfile

    ref_stubs.install()
    from cosmos_predict1.diffusion.module.pretrained_vae import VideoJITTokenizer

    out = {}
    with tempfile.TemporaryDirectory() as d:
        cases.write_tiny_tokenizer(d)
        x = cases.tiny_tokenizer_video()
        for tag, bf in (("f32", False), ("bf16", True)):
            tok = VideoJITTokenizer(name="tiny", latent_ch=16, is_bf16=bf, spatial_compression_factor=8,
                                    temporal_compression_factor=8, pixel_chunk_duration=17, max_enc_batch_size=1,
                                    max_dec_batch_size=1)
            tok.register_mean_std(d)
            tok.load_decoder(d)
            tok.load_encoder(d)
            z = tok.encode(x)
            y = tok.decode(z)
            out[f"z_{tag}"], out[f"y_{tag}"] = z.float().numpy(), y.float().numpy()
            out["frames"] = np.array([tok.get_latent_num_frames(1), tok.get_latent_num_frames(34), tok.get_pixel_num_frames(6),
                                      tok.latent_chunk_duration])
    golden.save(OUT, "vae_wrapper", **out)
    print("== tokenizer wrapper golden written: latent", out["z_f32"].shape, "video", out["y_f32"].shape, "==")
    return 0


def main():
    os.makedirs(OUT, exist_ok=True)
    only = sys.argv[1:]
    rc = 0
    if not only or "warp" in only:
        rc |= mint_warp()
    if not only or "classes" in only:
        rc |= mint_cache_classes()
    if not only or "dit" in only:
        rc |= mint_dit()
    if not only or "tokenizer" in only:
        rc |= mint_tokenizer()
    if not only or "fullwidth" in only:
        rc |= mint_dit_fullwidth()
    sys.exit(rc)


if __name__ == "__main__":
    main()
