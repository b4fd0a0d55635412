"""Host-side mirror of the reference's warp operators (Path R), backed by libgen3c_b200.so.

Same names, argument meaning and error behaviour as
``cosmos_predict1/diffusion/inference/forward_warp_utils_pytorch.py`` (reference file:line cited per
function).  Tensors are CUDA float32; there is no CPU path.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _lib

_workspaces: dict = {}


def _workspace(h: int, w: int, device: torch.device, max_items: int = 4):
    """One render workspace per (H, W, device): accumulation buffers for `max_items` frames.
    Under torch.use_deterministic_algorithms(True) it splats in the reference's fixed order (bitwise reproducible,
    as torch's index_put_(accumulate=True) is under that flag); otherwise with the faster float atomics."""
    key = (h, w, device.index, max_items)
    lib = _lib.load()
    ws = _workspaces.get(key)
    if ws is None:
        import ctypes as C

        handle = C.c_void_p()
        with torch.cuda.device(device):
            _lib.check(lib.g3c_render_create(h, w, max_items, C.byref(handle)), "g3c_render_create")
        ws = handle
        _workspaces[key] = ws
    with torch.cuda.device(device):
        _lib.check(lib.g3c_render_set_deterministic(ws, 1 if torch.are_deterministic_algorithms_enabled() else 0),
                   "g3c_render_set_deterministic")
    return ws


def _f32c(t: Optional[torch.Tensor], name: str) -> Optional[torch.Tensor]:
    if t is None:
        return None
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor (gen3c_b200 has no CPU path)")
    return t.to(torch.float32).contiguous()


def unproject_points(depth: torch.Tensor, w2c: torch.Tensor, intrinsic: torch.Tensor, is_depth: bool = True,
                     mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """reference :410-460.  depth (b,1,h,w), w2c (b,4,4), intrinsic (b,3,3) -> points (b,h,w,3)."""
    b, _, h, w = depth.shape
    depth = _f32c(depth, "depth")
    out = torch.empty((b, h, w, 3), device=depth.device, dtype=torch.float32)
    m8 = None
    if mask is not None:
        if mask.dim() == depth.dim() and mask.shape[1] == 1:
            mask = mask[:, 0]
        m8 = (mask != 0).to(torch.uint8).contiguous()
    lib = _lib.load()
    with torch.cuda.device(depth.device):
        _lib.check(lib.g3c_unproject_points(_lib.ptr(depth), _lib.ptr(_f32c(w2c, "w2c")),
                                            _lib.ptr(_f32c(intrinsic, "intrinsic")), _lib.ptr(m8), b, h, w,
                                            1 if is_depth else 0, _lib.ptr(out), _lib.stream_ptr()),
                   "g3c_unproject_points")
    return out


def reliable_depth_mask_range_batch(depth: torch.Tensor, window_size: int = 5, ratio_thresh: float = 0.05,
                                    eps: float = 1e-6) -> torch.Tensor:
    """reference :338-353 -> bool (b,1,h,w)."""
    assert window_size % 2 == 1, "Window size must be odd."
    if depth.dim() == 3:
        d = depth.unsqueeze(1)
    elif depth.dim() == 4:
        d = depth
    else:
        raise ValueError("depth tensor must be of shape (B, H, W) or (B, 1, H, W)")
    d = _f32c(d, "depth")
    b, _, h, w = d.shape
    out = torch.empty((b, 1, h, w), device=d.device, dtype=torch.uint8)
    lib = _lib.load()
    with torch.cuda.device(d.device):
        _lib.check(lib.g3c_reliable_depth_mask(_lib.ptr(d), b, h, w, window_size, ratio_thresh, eps, _lib.ptr(out),
                                               _lib.stream_ptr()), "g3c_reliable_depth_mask")
    return out.bool()


def bilinear_splatting(frame1: torch.Tensor, mask1: Optional[torch.Tensor], depth1: torch.Tensor,
                       flow12: torch.Tensor, flow12_mask: Optional[torch.Tensor] = None, is_image: bool = False,
                       n_views=1, depth_weight_scale=50) -> Tuple[torch.Tensor, torch.Tensor]:
    """reference :576-695 -> (warped (b,c,h,w), mask (b,1,h,w))."""
    if flow12_mask is not None or n_views != 1 or depth_weight_scale != 50:
        raise NotImplementedError("flow12_mask / n_views>1 / depth_weight_scale!=50 are not used by GEN3C inference")
    b, c, h, w = frame1.shape
    frame1 = _f32c(frame1, "frame1")
    out = torch.empty_like(frame1)
    mask2 = torch.empty((b, 1, h, w), device=frame1.device, dtype=torch.float32)
    lib = _lib.load()
    with torch.cuda.device(frame1.device):
        ws = _workspace(h, w, frame1.device)
        _lib.check(lib.g3c_bilinear_splatting(ws, _lib.ptr(frame1), _lib.ptr(_f32c(mask1, "mask1")),
                                              _lib.ptr(_f32c(depth1, "depth1")), _lib.ptr(_f32c(flow12, "flow12")),
                                              b, c, 1 if is_image else 0, _lib.ptr(out), _lib.ptr(mask2),
                                              _lib.stream_ptr()), "g3c_bilinear_splatting")
    return out, mask2


def splat_indices(flow12: torch.Tensor) -> torch.Tensor:
    """The integer destination indices of bilinear_splatting (reference :605-621):
    int32 (b,4,h,w) = floor_x, floor_y, ceil_x, ceil_y after clamping."""
    b, _, h, w = flow12.shape
    flow12 = _f32c(flow12, "flow12")
    idx = torch.empty((b, 4, h, w), device=flow12.device, dtype=torch.int32)
    lib = _lib.load()
    with torch.cuda.device(flow12.device):
        _lib.check(lib.g3c_splat_indices(_lib.ptr(flow12), b, h, w, _lib.ptr(idx), _lib.stream_ptr()),
                   "g3c_splat_indices")
    return idx


def forward_warp(
    frame1: torch.Tensor,
    mask1: Optional[torch.Tensor],
    depth1: Optional[torch.Tensor],
    transformation1: Optional[torch.Tensor],
    transformation2: torch.Tensor,
    intrinsic1: Optional[torch.Tensor],
    intrinsic2: Optional[torch.Tensor],
    is_image=True,
    conditioned_normal1=None,
    cameraray_filtering=False,
    is_depth=True,
    render_depth=False,
    world_points1=None,
    foreground_masking=False,
    boundary_mask=None,
) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor], torch.Tensor]:
    """reference :171-336.  Returns (warped_frame2, mask2, warped_depth2 | None, flow12)."""
    if conditioned_normal1 is not None or cameraray_filtering:
        raise NotImplementedError("normal / camera-ray filtering is not on the GEN3C inference path")
    if foreground_masking:
        assert boundary_mask is not None  # reference :286
    b, c, h, w = frame1.shape
    if intrinsic2 is None:
        assert intrinsic1 is not None, "intrinsic2 cannot be derived if intrinsic1 is None and intrinsic2 is None"
        intrinsic2 = intrinsic1.clone()
    if depth1 is None:
        assert world_points1.shape == (b, h, w, 3)
        points = _f32c(world_points1, "world_points1")
    else:
        assert mask1 is None or mask1.shape == (b, 1, h, w)
        assert depth1.shape == (b, 1, h, w)
        assert transformation1.shape == (b, 4, 4)
        assert transformation2.shape == (b, 4, 4)
        assert intrinsic1.shape == (b, 3, 3)
        assert intrinsic2.shape == (b, 3, 3)
        depth1 = torch.clamp(torch.nan_to_num(depth1, nan=1e4), min=0, max=1e4)
        # K2 (T2 T1^-1) (depth K1^-1 pix) == project(unproject(depth)); every pixel is unprojected
        points = unproject_points(depth1, transformation1, intrinsic1, is_depth=is_depth,
                                  mask=torch.ones_like(depth1, dtype=torch.uint8))
    frame1 = _f32c(frame1, "frame1")
    dev = frame1.device
    warped = torch.empty_like(frame1)
    mask2 = torch.empty((b, 1, h, w), device=dev, dtype=torch.float32)
    flow = torch.empty((b, 2, h, w), device=dev, dtype=torch.float32)
    want_depth = render_depth or foreground_masking
    depth2 = torch.empty((b, h, w), device=dev, dtype=torch.float32) if want_depth else None
    flags = (1 if want_depth else 0) | (0 if is_image else 2)
    lib = _lib.load()
    with torch.cuda.device(dev):
        ws = _workspace(h, w, dev)
        _lib.check(lib.g3c_forward_warp(ws, _lib.ptr(points), _lib.ptr(frame1), _lib.ptr(_f32c(mask1, "mask1")),
                                        _lib.ptr(_f32c(transformation2, "transformation2")),
                                        _lib.ptr(_f32c(intrinsic2, "intrinsic2")), b, c, flags, _lib.ptr(warped),
                                        _lib.ptr(mask2), _lib.ptr(depth2), _lib.ptr(flow), _lib.stream_ptr()),
                   "g3c_forward_warp")
        if foreground_masking:
            assert boundary_mask.shape == (b, h, w)
            bm = boundary_mask.to(device=dev, dtype=torch.uint8).contiguous()
            _lib.check(lib.g3c_foreground_occlusion(_lib.ptr(points), _lib.ptr(bm),
                                                    _lib.ptr(_f32c(transformation2, "transformation2")),
                                                    _lib.ptr(_f32c(intrinsic2, "intrinsic2")), b, c, h, w, _lib.ptr(warped),
                                                    _lib.ptr(mask2), _lib.ptr(depth2), _lib.stream_ptr()),
                       "g3c_foreground_occlusion")
    return warped, mask2, depth2, flow


def render_cache(points: torch.Tensor, images: torch.Tensor, masks: Optional[torch.Tensor], w2cs: torch.Tensor,
                 Ks: torch.Tensor, render_depth: bool = False, max_items_per_pass: int = 4,
                 boundary_masks: Optional[torch.Tensor] = None):
    """Fused cache render (the loop of reference cache_3d.py:175-223 in one native call).
    points (B,Fs,N,H,W,3), images (B,Fs,N,3,H,W), masks (B,Fs,N,1,H,W)|None, Fs in {1,F};
    w2cs (B,F,4,4), Ks (B,F,3,3) -> pixels (B,F,N,3,H,W) [depth (B,F,N,H,W) if render_depth], masks.
    boundary_masks (B,Fs,N,H,W) bool: foreground_masking=True — the mesh occlusion pass of forward_warp :285-335 runs
    on every item (a second native call) before the result is returned."""
    B, Fs, N, H, W, _ = points.shape
    F = w2cs.shape[1]
    dev = points.device
    fg = boundary_masks is not None
    pix = torch.empty((B, F, N, 3, H, W), device=dev, dtype=torch.float32)
    mk = torch.empty((B, F, N, 1, H, W), device=dev, dtype=torch.float32)
    dep = torch.empty((B, F, N, H, W), device=dev, dtype=torch.float32) if (render_depth or fg) else None
    lib = _lib.load()
    with torch.cuda.device(dev):
        ws = _workspace(H, W, dev, max_items_per_pass)
        pts, w2cs, Ks = _f32c(points, "points"), _f32c(w2cs, "w2cs"), _f32c(Ks, "Ks")
        _lib.check(lib.g3c_render_cache(ws, _lib.ptr(pts), _lib.ptr(_f32c(images, "images")),
                                        _lib.ptr(_f32c(masks, "masks")), _lib.ptr(w2cs), _lib.ptr(Ks), B, F, N, Fs,
                                        1 if dep is not None else 0, _lib.ptr(pix), _lib.ptr(mk), _lib.ptr(dep),
                                        _lib.stream_ptr()), "g3c_render_cache")
        if fg:
            assert boundary_masks.shape == (B, Fs, N, H, W)
            bm = boundary_masks.to(device=dev, dtype=torch.uint8).contiguous()
            _lib.check(lib.g3c_render_cache_occlusion(_lib.ptr(pts), _lib.ptr(bm), _lib.ptr(w2cs), _lib.ptr(Ks), B, F, N,
                                                      Fs, _lib.ptr(pix), _lib.ptr(mk), _lib.ptr(dep), H, W,
                                                      _lib.stream_ptr()), "g3c_render_cache_occlusion")
    return (dep if render_depth else pix), mk
