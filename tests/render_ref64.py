"""Float64 restatement of Path R (gen3c_b200/csrc/warp_render.cu) with a per-pixel error bound and a guard band.

Test infrastructure only.  The arithmetic is the reference's (oracle/warp_oracle.py cites the lines):
  project_points             q = K (w2c [p;1])[:3]
  forward_warp               m = mask * (q_z > 0),  flow = q_xy / (q_z + 1e-7) - grid
  bilinear_splatting         pos = flow + grid + 1, floor / ceil before clamping to [0, W+1] x [0, H+1],
                             w = frac * m / (exp(min(50 log1p(z) / (max log1p(z) + 1e-7), 80)) + 1e-7),
                             out = sum v w / sum w over the interior (the 1-px ring is cropped).

Positions are taken from a float32 flow (the kernel's own flow12 in the GPU tests), rounded exactly as the kernel
rounds them (fp32 adds), so the destination texels are the kernel's; everything after that is float64.

The bound.  out = sum v_i w_i / sum w_i.  If weight i carries a relative error of at most d_i, out moves by at most
about sum_i d_i w_i |v_i - out| / sum w (<= d_w max_i |v_i - out|, d_w = max d_i; doubled for second-order terms);
fp32 accumulation of n records adds (n + 3) u (sum |v_i| w_i / sum w_i + |out|), u = 2^-24.
d_w is derived per splat path (``path``):
  "exact"  (k_splat_points, the ordered splat of the deterministic mode):  IEEE expf / log1pf / divisions;
  "approx" (k_splat_points4):  log1p(z) = lg2.approx(1 + z) ln 2, ex2.approx, rcp.approx.  The log-depth error is
           multiplied by escale = 50 / lzmax, so this path loses accuracy in proportion to 1 / lzmax.

The guard band (texels excluded from the per-pixel check), computed from this reference alone:
  * knife edges: a texel that receives a record from a source whose position lies within KNIFE_ULP ulp of an integer
    (floor and ceil may flip there and the weight doubles), or whose projected depth is within its round-off of 0
    (the sign test q_z > 0 may flip);
  * tiny total weight: sum w < WFLOOR, below what fp32 resolves after the soft-z division.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
U = 2.0 ** -24          # fp32 unit round-off
KNIFE_ULP = 4           # positions this close (in ulp of the position) to an integer are knife edges
WFLOOR = 1e-30          # total weights below this are not resolved in fp32
# hardware approximations of k_splat_points4 (PTX ISA: lg2.approx, ex2.approx max error ~2^-22; rcp.approx 1 ulp)
LG2_ABS = 2.0 ** -22
EX2_REL = 2.0 ** -22
RCP_REL = 2.0 ** -23


def project64(points, w2c, K):
    """points (H, W, 3), w2c (4, 4), K (3, 3) -> q (H, W, 3) in float64 and a bound on |q32 - q| per component.
    The bound: each fp32 fma/add of the kernel's chain rounds once, so |error| <= 4 u sum |terms| per camera-space
    component, propagated through K with another 3 u."""
    p = points.astype(np.float64)
    M = w2c.astype(np.float64)
    k = K.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        cam = p @ M[:3, :3].T + M[:3, 3]
        cabs = np.abs(p) @ np.abs(M[:3, :3]).T + np.abs(M[:3, 3])
        q = cam @ k.T
        qerr = (4 * U * cabs) @ np.abs(k).T + 3 * U * (np.abs(cam) @ np.abs(k).T)
    return q, qerr


def flow64(q, qerr, H, W):
    """flow = q_xy / (q_z + 1e-7) - grid in float64, with a bound on the kernel's fp32 flow: the propagated projection
    error plus the roundings of the add, the division and the subtraction."""
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        den = q[..., 2] + 1e-7
        r = q[..., :2] / den[..., None]
        fl = np.stack([r[..., 0] - xs, r[..., 1] - ys])
        rerr = (qerr[..., :2] + np.abs(r) * (qerr[..., 2:3] + U * np.abs(den)[..., None])) / np.abs(den)[..., None]
        ferr = np.moveaxis(rerr + 2 * U * np.abs(r), -1, 0) + U * np.abs(fl)
    return fl, ferr


def positions32(flow32, H, W):
    """The kernel's fp32 positions (flow + x) + 1 and the clamped floor / ceil indices (splat_indices)."""
    ys, xs = np.mgrid[0:H, 0:W].astype(F32)
    with np.errstate(invalid="ignore", over="ignore"):
        pos = np.stack([(flow32[0].astype(F32) + xs) + F32(1), (flow32[1].astype(F32) + ys) + F32(1)])
    lim = np.array([W + 1, H + 1], np.float64).reshape(2, 1, 1)
    p64 = np.nan_to_num(pos.astype(np.float64), nan=0.0, posinf=1e30, neginf=-1e30)
    fl = np.clip(np.floor(p64), 0, lim)
    ce = np.clip(np.ceil(p64), 0, lim)
    pc = np.clip(p64, 0, lim)
    return pos, pc, fl.astype(np.int64), ce.astype(np.int64)


def lz_error(z, zerr, path):
    """Bound on |lz32 - log1p(max(z, 0))| for the two log-depth evaluations."""
    zc = np.maximum(z, 0)
    lz = np.log1p(zc)
    base = zerr / (1 + zc) + 2 * U * lz
    if path == "exact":
        return base
    # lg2.approx(1 + z) ln 2: rounding of 1 + z, the approximation's absolute error, the ln 2 multiply
    return base + U + np.log(2) * LG2_ABS * (1 + np.abs(np.log2(1 + zc))) + U * lz


def splat(frame, mask, z, flow32, lzmax, zerr=None, path="exact", is_image=True, lzmax_err=0.0, pos_err=None,
          swap_ne_sw=False, soft_z=True, crop_shift=0, ignore_mask=False):
    """One item.  frame (C, H, W), mask (H, W) | None, z (H, W) float64 projected depth, flow32 (2, H, W) float32,
    lzmax the group's float64 max of log1p(max(z, 0)).  Returns a dict of per-texel arrays (H, W):
      out (C, H, W), mask, depth (sum z w / sum w), sw (sum w), n (records), dev (max |v_i - out|, per channel
      maximum), sabs (sum |v| w / sum w), dw (largest relative weight error of the texel's records), guard (bool),
      bound (C, H, W) and dbound (depth).
    pos_err (2, H, W): when the positions are another implementation's estimate rather than the checked one's own,
    the distance they may be off by; it widens the knife edges and adds pos_err / frac to each weight's error.
    The keyword switches after ``lzmax_err`` build the negative controls (ignored by the product)."""
    C, H, W = frame.shape
    HW = H * W
    zerr = np.zeros_like(z) if zerr is None else zerr
    m = np.ones((H, W)) if (mask is None or ignore_mask) else mask.astype(np.float64)
    with np.errstate(invalid="ignore"):
        m = m * (z > 0)
    pos, pc, fl, ce = positions32(flow32, H, W)
    frac_f = 1 - (pc - fl)          # (2, H, W): x, y
    frac_c = 1 - (ce - pc)
    zc = np.maximum(np.nan_to_num(z, nan=0.0), 0)
    lz = np.log1p(zc)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        e = lz / (lzmax + 1e-7) * 50.0 if soft_z else np.zeros_like(lz)
        e = np.fmin(e, 80.0)        # fminf: a NaN exponent (lz = lzmax = inf) becomes 80
        dwt = np.exp(e) + 1e-7
    # relative weight error of each source
    lze = lz_error(zc, zerr, path)
    escale = 50.0 / (lzmax + 1e-7)
    with np.errstate(invalid="ignore"):
        de = escale * lze + np.nan_to_num(e) * (lzmax_err / max(lzmax, 1e-30) + 3 * U)
    if path == "exact":
        dwr = de + 2 * U + 4 * U
    else:
        dwr = de + EX2_REL + RCP_REL + np.nan_to_num(e) * U + 4 * U
    corners = [("nw", frac_f[1] * frac_f[0], fl[1], fl[0]), ("sw", frac_c[1] * frac_f[0], ce[1], fl[0]),
               ("ne", frac_f[1] * frac_c[0], fl[1], ce[0]), ("se", frac_c[1] * frac_c[0], ce[1], ce[0])]
    if swap_ne_sw:
        corners[1], corners[2] = (("sw", corners[2][1], corners[1][2], corners[1][3]),
                                  ("ne", corners[1][1], corners[2][2], corners[2][3]))
    # knife edges: a position within KNIFE_ULP ulp of an integer, or a depth whose sign is uncertain
    with np.errstate(invalid="ignore"):
        dpos = KNIFE_ULP * np.spacing(np.abs(pos)).astype(np.float64)
        if pos_err is not None:
            dpos = dpos + pos_err
        near = np.abs(pos.astype(np.float64) - np.round(pos.astype(np.float64))) <= dpos
    knife = near[0] | near[1] | (np.abs(np.nan_to_num(z, nan=0.0)) <= zerr)
    v = frame.reshape(C, HW).astype(np.float64)
    zz = np.nan_to_num(z, nan=0.0).reshape(HW)
    recs = []
    rel = []
    for ci, (_, fw, ty, tx) in enumerate(corners):
        d_i = dwr
        if pos_err is not None:
            fx_, fy_ = (frac_f if ci in (0, 1) else frac_c)[0], (frac_f if ci in (0, 2) else frac_c)[1]
            with np.errstate(divide="ignore", invalid="ignore"):
                d_i = dwr + pos_err[0] / fx_ + pos_err[1] / fy_
        rel.append(np.nan_to_num(d_i, nan=np.inf).reshape(HW))
        with np.errstate(invalid="ignore", over="ignore"):
            w = (fw * m / dwt).reshape(HW)
        ty = ty.reshape(HW) - 1
        tx = tx.reshape(HW) - 1 + crop_shift
        keep = (w != 0) & (ty >= 0) & (ty < H) & (tx >= 0) & (tx < W)
        idx = np.where(keep, ty * W + np.clip(tx, 0, W - 1), -1)
        recs.append((idx, np.where(keep, w, 0.0)))
    idx = np.concatenate([r[0] for r in recs])
    wts = np.concatenate([r[1] for r in recs])
    rel = np.concatenate(rel)
    src = np.tile(np.arange(HW), 4)
    sel = idx >= 0
    idx, wts, src, rel = idx[sel], wts[sel], src[sel], rel[sel]
    sw = np.bincount(idx, wts, HW)
    n = np.bincount(idx, None, HW)
    acc = np.stack([np.bincount(idx, wts * v[c, src], HW) for c in range(C)])
    sabs = np.stack([np.bincount(idx, wts * np.abs(v[c, src]), HW) for c in range(C)])
    accz = np.bincount(idx, wts * zz[src], HW)
    hit = sw > 0
    with np.errstate(invalid="ignore", divide="ignore"):
        raw = np.where(hit, acc / np.where(hit, sw, 1), 0.0)
        depth = np.where(hit, accz / np.where(hit, sw, 1), 0.0)
        sabs = np.where(hit, sabs / np.where(hit, sw, 1), 0.0)
    dev = np.zeros((C, HW))
    for c in range(C):
        np.maximum.at(dev[c], idx, np.abs(v[c, src] - raw[c, idx]))
    ddev = np.zeros(HW)
    np.maximum.at(ddev, idx, np.abs(zz[src] - depth[idx]))
    dwmax = np.zeros(HW)
    np.maximum.at(dwmax, idx, rel)
    # first order: |d out| <= sum_i d_i w_i |v_i - out| / sum w (doubled for the second-order terms)
    with np.errstate(invalid="ignore", divide="ignore"):
        wsum1 = np.where(hit, sw, 1)
        pert = np.stack([np.bincount(idx, np.minimum(rel, 1.0) * wts * np.abs(v[c, src] - raw[c, idx]), HW) / wsum1
                         for c in range(C)])
        dpert = np.bincount(idx, np.minimum(rel, 1.0) * wts * np.abs(zz[src] - depth[idx]), HW) / wsum1
    zemax = np.zeros(HW)
    np.maximum.at(zemax, idx, zerr.reshape(HW)[src])
    kn = np.zeros(HW, bool)
    kn[idx[knife.reshape(HW)[src]]] = True
    tiny = hit & (sw < WFLOOR)
    guard = kn | tiny
    fill = -1.0 if is_image else 0.0
    out = np.where(hit, raw, fill)
    if is_image:
        out = np.clip(out, -1, 1)
    bound = 2 * pert + (n + 3) * U * (sabs + np.abs(raw))
    dbound = 2 * dpert + (n + 3) * U * 2 * np.abs(depth) + zemax
    r = dict(out=out, mask=hit.astype(np.float64), depth=depth, sw=sw, n=n, dev=dev, sabs=sabs, dw=dwmax,
             guard=guard, tiny=tiny, bound=bound, dbound=dbound)
    return {k: (a.reshape((C, H, W)) if a.ndim == 2 else a.reshape(H, W)) for k, a in r.items()}


def group_lzmax(zs, zerrs):
    """The group's log-depth max (over every pixel, mask or not, like k_project_max) and a bound on its error.
    NaN depths are dropped (fmaxf(NaN, 0) = 0 in log_depth)."""
    zc = [np.maximum(np.nan_to_num(z, nan=0.0), 0) for z in zs]
    lz = np.max([np.log1p(z).max() for z in zc])
    err = max(float(np.max(e / (1 + z) + 2 * U * np.log1p(z))) for z, e in zip(zc, zerrs))
    return lz, err


def forward_warp(frames, masks, points, w2cs, Ks, flows32, path, is_image=True, group=None, foreign_flow=False, **ctl):
    """Items of one or more groups (``group`` consecutive items share a max; default: all of them, forward_warp's
    group = b).  frames (b, C, H, W), masks (b, H, W) | None, points (b, H, W, 3), flows32 (b, 2, H, W) from the
    kernel.  Returns a list of per-item dicts of ``splat`` plus the float64 flow, its bound and the depth."""
    b = frames.shape[0]
    group = b if group is None else group
    H, W = frames.shape[2:]
    proj = [project64(points[i], w2cs[i], Ks[i]) for i in range(b)]
    res = []
    for g0 in range(0, b, group):
        items = range(g0, min(g0 + group, b))
        lzmax, lerr = group_lzmax([proj[i][0][..., 2] for i in items], [proj[i][1][..., 2] for i in items])
        for i in items:
            q, qe = proj[i]
            lzm, le = lzmax, lerr
            if ctl.get("per_item_max"):
                lzm, le = group_lzmax([q[..., 2]], [qe[..., 2]])
            kw = {k: v for k, v in ctl.items() if k != "per_item_max"}
            f64, ferr = flow64(q, qe, H, W)
            if foreign_flow:   # flows32 comes from another fp32 evaluation of the projection: both may be off by ferr
                kw["pos_err"] = 2 * np.nan_to_num(ferr, nan=np.inf)
            r = splat(frames[i], None if masks is None else masks[i], q[..., 2], flows32[i], lzm, qe[..., 2], path,
                      is_image, le, **kw)
            r["flow"], r["flow_err"] = f64, ferr
            r["z"], r["zerr"] = q[..., 2], qe[..., 2]
            res.append(r)
    return res


def excess(x, ref, bound, guard):
    """max over non-guarded texels of |x - ref| / bound (<= 1 passes); x, ref, bound (..., H, W), guard (H, W)."""
    keep = np.broadcast_to(~guard, x.shape)
    d = np.abs(x.astype(np.float64) - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d == 0, 0.0, d / np.maximum(bound, 1e-300))
    return float(r[keep].max()) if keep.any() else 0.0


# ---------------------------------------------------------------------------------------------------------------------
# unproject, reliability mask, depth alignment
# ---------------------------------------------------------------------------------------------------------------------
def unproject64(depth, w2c, K, is_depth=True, mask=None):
    """depth (H, W) -> (points (H, W, 3), bound).  Points of invalid pixels are 0 (valid = mask, or depth > 0).
    The bound: the kernel inverts K and w2c in double and rounds them to fp32 (u relative per entry), then evaluates
    the fp32 chain; 8 u of the absolute sums of every stage, and 4 u |p| for the normalisation of rays."""
    H, W = depth.shape
    kinv = np.linalg.inv(K.astype(np.float64))
    c2w = np.linalg.inv(w2c.astype(np.float64))
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    pix = np.stack([xs, ys, np.ones_like(xs)], -1)
    ray = pix @ kinv.T
    rabs = pix @ np.abs(kinv).T
    d = depth.astype(np.float64)[..., None]
    if not is_depth:
        nrm = np.linalg.norm(ray, axis=-1, keepdims=True) + 1e-8
        ray = ray / nrm
        rabs = rabs / nrm + 6 * U * np.abs(ray)
    cam = d * ray
    cabs = np.abs(d) * rabs
    p = cam @ c2w[:3, :3].T + c2w[:3, 3]
    bound = 8 * U * (cabs @ np.abs(c2w[:3, :3]).T + np.abs(c2w[:3, 3]) + np.abs(cam) @ np.abs(c2w[:3, :3]).T)
    valid = (depth > 0) if mask is None else mask.astype(bool)
    p = np.where(valid[..., None], p, 0.0)
    return p, np.where(valid[..., None], bound, 0.0), valid


def reliable64(depth, window, thresh, eps=1e-6):
    """depth (H, W) -> (mask, guard): max / min pools ignore the padding, the mean counts zeros over window^2.
    guard: the float64 ratio lies within its fp32 round-off of the threshold."""
    H, W = depth.shape
    d = depth.astype(np.float64)
    r = window // 2
    mx = np.full((H, W), -np.inf)
    mn = np.full((H, W), np.inf)
    sm = np.zeros((H, W))
    sabs = np.zeros((H, W))
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            if abs(dy) >= H or abs(dx) >= W:
                continue
            ys, xs = slice(max(0, -dy), H - max(0, dy)), slice(max(0, -dx), W - max(0, dx))
            yo, xo = slice(max(0, dy), H - max(0, -dy)), slice(max(0, dx), W - max(0, -dx))
            mx[ys, xs] = np.maximum(mx[ys, xs], d[yo, xo])
            mn[ys, xs] = np.minimum(mn[ys, xs], d[yo, xo])
            sm[ys, xs] += d[yo, xo]
            sabs[ys, xs] += np.abs(d[yo, xo])
    mean = sm / (window * window)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = (mx - mn) / (mean + eps)
        rerr = np.abs(ratio) * ((window * window + 3) * U * sabs / (window * window) / np.abs(mean + eps) + 3 * U)
    mask = (ratio < thresh) & (d > 0)
    guard = (np.abs(ratio - thresh) <= rerr + U * thresh) & (d > 0)
    return mask, guard


def box3(a):
    H, W = a.shape
    p = np.pad(a, 1)
    return sum(p[dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)) / 9.0


def align64(depth, target, tmask, K, c2w, num_iters, lambda_arap=0.1, lr=1e-3, drop_bias=None):
    """The non-rigid depth alignment (warp_render.cu k_align_*; oracle warp_oracle.align_depth after the rigid fit) in
    float64: sc = 1, num_iters Adam steps on the closed-form gradient
        coef_p sign(d_p sc_p - t_p) + a_w (box3(g) - g),  g = sign(box3(sc) - sc)  (zero padding),  a_w = lambda / (H W),
    coef_p = mask_p d_p |R K^-1 (x, y, 1)|_1 / (3 max(n, 1)).  Returns (depth * sc, tol, guard).

    Sign ties of the smoothness term are structural: the first Adam steps move every pixel by the same +-lr, so
    neighbourhoods of equal sc are common, and fp32's box3 of equal values differs from the value by +-1 ulp for about
    half of them (nine fmas with fl(1/9); only box3 of 1.0 is exact).  So the check splits the pixels:
      * data pixels (coef_p >= 16 a_w): whatever the smoothness signs, |box3(g) - g| <= 2, so they move the gradient by
        at most rho = 4 a_w / coef_p relative and Adam's update (|update| <= ~3.2 lr) by 2 rho of it.  tol adds that per
        step; the guard holds the pixels whose data residual d sc - t came within tol or round-off of 0;
      * smoothness pixels (the rest): a tie within their 3x3 neighbourhood, or a guarded pixel within 2 px per later
        step, guards them.
    Both carry the fp32 round-off of the updates, 16 u per step.  ``drop_bias`` in {"m1", "m2"} drops one Adam bias
    correction (negative control)."""
    H, W = depth.shape
    d = depth.astype(np.float64)
    t = target.astype(np.float64)
    mask = tmask.astype(bool)
    n = int(mask.sum())
    kinv = np.linalg.inv(K.astype(np.float64))
    rot = np.linalg.inv(c2w.astype(np.float64))[:3, :3]
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    rays = np.stack([xs, ys, np.ones_like(xs)], -1) @ kinv.T
    coef = np.where(mask, d * np.abs(rays @ rot.T).sum(-1) / (3 * max(n, 1)), 0.0)
    aw = lambda_arap / (H * W)
    strong = coef >= 16 * aw
    with np.errstate(divide="ignore"):
        rho = np.where(strong, 4 * aw / np.where(strong, coef, 1.0), 0.0)
    sc = np.ones((H, W))
    m1 = np.zeros((H, W))
    m2 = np.zeros((H, W))
    tol_sc = np.full((H, W), 2 * U)
    guard = np.zeros((H, W), bool)
    inner = np.zeros((H, W), bool)
    if H > 2 and W > 2:
        inner[1:-1, 1:-1] = True

    def dilate(g, r):
        for _ in range(r):
            g = box3(g.astype(np.float64)) > 0
        return g

    for it in range(1, num_iters + 1):
        e = d * sc - t
        etie = np.abs(e) <= d * tol_sc + 8 * U * (np.abs(d * sc) + np.abs(t))
        a = box3(sc) - sc
        flat = np.abs(a) <= 16 * U * box3(np.abs(sc))
        ones = (box3((sc == 1.0).astype(np.float64)) >= 1 - 1e-12) & inner     # box3 of 1.0 is exact in fp32
        g = np.where(flat, 0.0, np.sign(a))
        guard = np.where(strong, guard | etie, dilate(guard, 2) | etie | dilate(flat & ~ones, 1))
        grad = coef * np.where(etie, 0.0, np.sign(e)) + aw * (box3(g) - g)
        m1 = 0.9 * m1 + 0.1 * grad
        m2 = 0.999 * m2 + 0.001 * grad * grad
        step = lr / (1 - 0.9 ** it) if drop_bias != "m1" else lr
        bc2 = np.sqrt(1 - 0.999 ** it) if drop_bias != "m2" else 1.0
        sc = sc - step * m1 / (np.sqrt(m2) / bc2 + 1e-8)
        tol_sc = tol_sc + 2 * rho * 3.2 * lr + 16 * U
    return d * sc, d * tol_sc, guard
