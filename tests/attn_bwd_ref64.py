"""Float64 restatement of the attention backward (gen3c_b200/csrc/attn_bwd_wgmma.cu) with a per-element error bound
and a per-(row, head) statistical bar, in the manner of tests/attn_ref64.py.

Test infrastructure only.  Per head (128 dims), with x_ik = (q_i . k_k) sl2 (log2 units, sl2 as in attn_ref64), the
forward's lse_i = log2 sum_k 2^x_ik, P = 2^(x - lse), o64 = P v, the kernels compute

    Delta_i = fp32 sum_d dO_id O_id             (O: the forward's bf16 output)
    P~_ik   = ex2.approx.ftz(fma(s_ik, sl2, -lse~_i))   (s from wgmma, lse~ the forward's fp32 lse)
    dS~_ik  = P~_ik (dP~_ik - Delta_i),          dP~ = dO v^T from wgmma
    dV = sum_i bf16(P~_ik) dO_i,  dQ = scale sum_k bf16(dS~_ik) k_k,  dK = scale sum_i bf16(dS~_ik) q_i

(fp32 accumulation), and the reference evaluates dV64 = P^T dO, dS = P o (dO v^T - Delta64), Delta64 = sum_d dO o64,
dQ64 = scale dS k, dK64 = scale dS^T q in float64 from the exact bf16 inputs.  The gradient factor is `scale` as passed
(the kernels' convention); with scale = ln 2 and sl2 = 1 this is the derivative of 2^x up to fp32(ln 2).

The per-element bound is MARGIN times the sum of these terms (eps_ik is the relative error of P~_ik, capped at 1):
  * score, fma argument and ex2.approx:  eta_ik = ln 2 (sl2 S_REL sum_d |q_id k_kd| + 2^-24 |x_ik - lse_i|) + 2^-22,
    the same model as the forward's (a 128-term wgmma product, one rounding of the exponent's argument);
  * the forward's lse error (common to a row):  ln 2 dlse_i with dlse_i = (sum_k P_ik eta'_ik + (16 n_kv + 8) 2^-24)
    / ln 2 + 2^-22 (|lse_i| + 32), eta' the forward's eta (m trails the row max by up to 24 under the sum guard), the
    fp32 sum l over n_kv tiles, and the fp32 m + log2(l);  eps = eta + ln 2 dlse;
  * dP from wgmma:  S_REL sum_d |dO_id v_kd|;
  * Delta from the bf16 O instead of o64:  eD_i = sum_d |dO_id| Bo_d + 2^-24 128 sum_d |dO_id o64_d|, Bo the forward's
    per-element bound of attn_ref64 (its MARGIN included) plus the fp32 summation of the 128 products;
  so |dS~ - dS| <= e_dS = P eps |dP - Delta| + P (1 + eps) (S_REL sum |dO v| + eD);
  * the bf16 rounding of P and dS inside the MMAs:  2^-8 (P (1 + eps)) and 2^-8 (|dS| + e_dS) per term;
  * fp32 accumulation over Lq (dK, dV: 16 roundings per 128 queries, as 4 k-steps per 64-query step) or Lk (dQ):
    (16 ceil(L / 64) + 8) 2^-24 times the sum of the absolute terms;
  * flushed exponentials (ex2.approx.ftz):  L 2^-118 times the largest operand row;
  * the final multiply by scale (one fp32 rounding) and the output rounding (one bf16 spacing at |g64|).
Every term is a worst case; MARGIN = 2 covers the second-order products left out (e.g. eps times 2^-8) with room.

The statistical bar closes the gap of diffuse rows, where the 2^-8 terms grow like the sum of absolute values and the
actual error like its root-sum-square.  A (row, head) is diffuse when its largest term (|dS| for dQ and dK, P for dV)
is at most DIFFUSE = 1/32 of the sum of its terms; rows led by a few terms, whose errors need not be independent, are
held to the element bound alone (it is tight there).  The error norm over the 128 dims of a diffuse row must be at
most SIGMA_BAR sigma + the norm of the row-coherent part.  Inputs built from a few repeated directions (rows of
+-250 logits along one vector) make the roundings of different terms equal rather than independent: they are held to
the element bound alone (check(stat=False)).  sigma^2 sums, per element, independent
errors of each term: the bf16 roundings of P and dS (variance at most (2^-16 / 3) t^2 for a term t), the score and ex2
errors taken as independent per term and uniform within +-eta (variance eta^2 t^2 / 3), the Delta error of each query
row (independent between rows, variance from the forward's roundings of O: spacing^2 / 12 and (2^-16 / 3) sum_j
P_ij^2 v_jd^2 per dim), and the output rounding (spacing^2 / 12).  The row-coherent part is the forward's lse error in
dQ (it scales every P of a query row alike: ln 2 dlse_i |dQ64_i|) and, in dQ, the Delta error of that row (variance
varD_i (P k)_d^2, kept inside sigma).  A dropped 128-key or 64-query tile moves a diffuse row by tens of sigma.
"""
from __future__ import annotations

import torch

from tests.attn_ref64 import ACC_C, ACC_PER_TILE, BF16_P, EX2_REL, FLUSH, LN2, S_REL, TILE, U, bf16_spacing, scale_log2

MARGIN = 2.0
SIGMA_BAR = 6.0
DIFFUSE = 1.0 / 32
GUARD_LAG = 24.0  # how far the forward's reference m may trail the row max (log2 units, sum guard of attn_wgmma.cu)


def _acc(L: int) -> float:
    """fp32 accumulation roundings (relative) over L terms fed 16 per k-step, 64 per dK/dV step."""
    return (ACC_PER_TILE * ((L + 63) // 64) + ACC_C) * U


class BwdReference:
    """float64 gradients, bounds and sigmas of one attention backward.

    q [Lq, heads*128], k and v [Lk, heads*128], dout [Lq, heads*128] (token-major, any dtype / device; evaluated in
    float64 where they are).  q_rows / k_rows select the rows of dQ and of dK, dV that are evaluated (all when None);
    dK and dV rows always sum over every query.  Attributes dq, dk, dv (float64) and bq, bk, bv (bounds) of the
    selected rows, and sq, sk, sv [rows, heads] (sigma) with cq [rows, heads] (row-coherent norm of dQ)."""

    def __init__(self, q, k, v, dout, heads, scale, q_rows=None, k_rows=None, block=512):
        self.sl2 = sl2 = scale_log2(scale)
        self.scale = scale
        self.heads = heads
        Lq, Lk = q.shape[0], k.shape[0]
        n_kv = (Lk + TILE - 1) // TILE
        dev = q.device
        f64 = torch.float64
        q_idx = torch.arange(Lq, device=dev) if q_rows is None else torch.as_tensor(q_rows, device=dev)
        k_idx = torch.arange(Lk, device=dev) if k_rows is None else torch.as_tensor(k_rows, device=dev)
        Rq, Rk = len(q_idx), len(k_idx)
        self.dq = torch.zeros(Rq, heads * 128, dtype=f64, device=dev)
        self.bq, self.dk, self.bk, self.dv, self.bv = (torch.zeros(Rk if i else Rq, heads * 128, dtype=f64, device=dev)
                                                       for i in (0, 1, 1, 1, 1))
        self.sq = torch.zeros(Rq, heads, dtype=f64, device=dev)
        self.cq = torch.zeros(Rq, heads, dtype=f64, device=dev)
        self.sk, self.sv = (torch.zeros(Rk, heads, dtype=f64, device=dev) for _ in range(2))
        # largest term's share of the summed |terms| of each row (|dS| for dQ, dK; P for dV): the bar applies to the
        # rows where it is at most DIFFUSE
        self.fq = torch.ones(Rq, heads, dtype=f64, device=dev)
        self.fk, self.fv = (torch.ones(Rk, heads, dtype=f64, device=dev) for _ in range(2))
        acc_q, acc_kv = _acc(Lk), _acc(Lq)
        for h in range(heads):
            hs = slice(h * 128, (h + 1) * 128)
            kh, vh = k[:, hs].to(f64), v[:, hs].to(f64)
            kabs, vabs = kh.abs(), vh.abs()
            vmax = float(vabs.max())
            # dK / dV rows k_idx: accumulated over query blocks
            dk = torch.zeros(Rk, 128, dtype=f64, device=dev)
            dv, ek, ev, vk, vv = (torch.zeros_like(dk) for _ in range(5))
            mk, sk, mv, sv = (torch.zeros(Rk, dtype=f64, device=dev) for _ in range(4))  # largest / summed |terms|
            for r0 in range(0, Lq, block):
                st = self._rows(q[r0:r0 + block, hs].to(f64), dout[r0:r0 + block, hs].to(f64), kh, vh, kabs, vabs,
                                vmax, n_kv, k_idx)
                qb, dob = st["q"], st["do"]
                P, dS, eP, edS, eta_t, eDv = st["P"], st["dS"], st["eP"], st["edS"], st["edS_rand"], st["varD"]
                dk += dS.T @ qb
                dv += P.T @ dob
                mk = torch.maximum(mk, dS.abs().amax(0))
                mv = torch.maximum(mv, P.amax(0))
                sk += dS.abs().sum(0)
                sv += P.sum(0)
                # bounds (before scale / margin): dV from P, dK from dS
                ev += (eP + BF16_P * (P + eP)).T @ dob.abs() + acc_kv * (P.T @ dob.abs())
                ek += (edS + BF16_P * (dS.abs() + edS)).T @ qb.abs() + acc_kv * (dS.abs().T @ qb.abs())
                # variances
                vv += (2.0 ** -16 / 3) * ((P * P).T @ (dob * dob)) + ((st["eP_rand"] ** 2) / 3).T @ (dob * dob)
                vk += ((2.0 ** -16 / 3) * (dS * dS) + eta_t ** 2 / 3 + P * P * eDv[:, None]).T @ (qb * qb)
            dk *= scale
            flush_k = Lq * FLUSH * float(dout[:, hs].abs().max()) * (vmax + 1.0)
            spk, spv = bf16_spacing(dk), bf16_spacing(dv)
            self.dk[:, hs], self.dv[:, hs] = dk, dv
            self.bk[:, hs] = MARGIN * (scale * ek * (1 + 2 * U) + U * dk.abs() + flush_k * float(q[:, hs].abs().max())
                                       + spk)
            self.bv[:, hs] = MARGIN * (ev + Lq * FLUSH * float(dout[:, hs].abs().max()) + spv)
            self.sk[:, h] = (scale * scale * vk + spk * spk / 12).sum(1).sqrt()
            self.sv[:, h] = (vv + spv * spv / 12).sum(1).sqrt()
            self.fk[:, h], self.fv[:, h] = mk / sk.clamp_min(1e-300), mv / sv.clamp_min(1e-300)
            # dQ rows q_idx
            for r0 in range(0, Rq, block):
                rows = q_idx[r0:r0 + block]
                st = self._rows(q[rows][:, hs].to(f64), dout[rows][:, hs].to(f64), kh, vh, kabs, vabs, vmax, n_kv,
                                None)
                P, dS, edS = st["P"], st["dS"], st["edS"]
                dq = scale * (dS @ kh)
                eq = (edS + BF16_P * (dS.abs() + edS)) @ kabs + acc_q * (dS.abs() @ kabs)
                sp = bf16_spacing(dq)
                flush_q = Lk * FLUSH * (vmax + 1.0) * float(dout[:, hs].abs().max()) * float(kabs.max())
                self.dq[r0:r0 + block, hs] = dq
                self.bq[r0:r0 + block, hs] = MARGIN * (scale * eq * (1 + 2 * U) + U * dq.abs() + flush_q + sp)
                var = (scale * scale * ((2.0 ** -16 / 3) * ((dS * dS) @ (kh * kh)) + (st["edS_rand"] ** 2 / 3) @ (kh * kh)
                                        + st["varD"][:, None] * (P @ kh) ** 2) + sp * sp / 12)
                self.sq[r0:r0 + block, h] = var.sum(1).sqrt()
                self.cq[r0:r0 + block, h] = MARGIN * (LN2 * st["dlse"][:, None] * dq.abs()).norm(dim=1)
                self.fq[r0:r0 + block, h] = dS.abs().amax(1) / dS.abs().sum(1).clamp_min(1e-300)

    def _rows(self, qb, dob, kh, vh, kabs, vabs, vmax, n_kv, cols):
        """Everything a block of query rows contributes; P, dS and their errors restricted to the keys `cols`."""
        sl2 = self.sl2
        x = (qb @ kh.T) * sl2
        mx = x.amax(1, keepdim=True)
        p = torch.exp2(x - mx)
        lsum = p.sum(1, keepdim=True)
        lse = mx + torch.log2(lsum)
        w = p / lsum
        o = w @ vh
        A = w @ vabs
        qk = qb.abs() @ kabs.T
        # forward: eta' (m up to GUARD_LAG below the row max), its output bound Bo (attn_ref64) and variance
        eta_f = (LN2 * (sl2 * S_REL * qk + U * ((x - mx).abs() + GUARD_LAG)) + EX2_REL).clamp(max=1.0)
        we = w * eta_f
        pert = we @ vabs + we.sum(1, keepdim=True) * o.abs()
        acc_f = (ACC_PER_TILE * n_kv + ACC_C) * U + n_kv * EX2_REL
        sp_o = bf16_spacing(o)
        Bo = 2.0 * (BF16_P * A + 2 * pert + acc_f * (A + o.abs()) + kh.shape[0] * FLUSH * vmax + sp_o)
        var_o = (2.0 ** -16 / 3) * ((w * w) @ (vh * vh)) + sp_o * sp_o / 12
        dlse = (we.sum(1) + ((ACC_PER_TILE * n_kv + ACC_C) * U)) / LN2 + EX2_REL * (lse[:, 0].abs() + 32.0)
        delta = (dob * o).sum(1)
        eD = (dob.abs() * Bo).sum(1) + 128 * U * (dob * o).abs().sum(1)
        varD = ((dob * dob) * var_o).sum(1)
        if cols is not None:
            x, w, qk, vc, vabs_c = x[:, cols], w[:, cols], qk[:, cols], vh[cols], vabs[cols]
        else:
            vc, vabs_c = vh, vabs
        P = w
        dP = dob @ vc.T
        G = dP - delta[:, None]
        dS = P * G
        eta = (LN2 * (sl2 * S_REL * qk + U * (x - lse).abs()) + EX2_REL).clamp(max=1.0)
        eps = (eta + LN2 * dlse[:, None]).clamp(max=1.0)
        e_dP = S_REL * (dob.abs() @ vabs_c.T)
        eP = P * eps
        edS = eP * G.abs() + P * (1 + eps) * (e_dP + eD[:, None])
        return dict(q=qb, do=dob, P=P, dS=dS, eP=eP, edS=edS, eP_rand=P * eta,
                    edS_rand=P * eta * G.abs() + P * e_dP, varD=varD, dlse=dlse)

    def ratios(self, dq=None, dk=None, dv=None):
        """{name: (largest |g - g64| / bound, largest error norm / bar over (row, head), (row, head) of the latter)}
        for the gradients given (the rows of this reference, in its row order)."""
        out = {}
        for name, g, ref, bnd, sig, coh, fr in (("dq", dq, self.dq, self.bq, self.sq, self.cq, self.fq),
                                                ("dk", dk, self.dk, self.bk, self.sk, None, self.fk),
                                                ("dv", dv, self.dv, self.bv, self.sv, None, self.fv)):
            if g is None:
                continue
            d = g.double().to(ref.device) - ref
            e = float((d.abs() / bnd).max()) if d.numel() else 0.0
            n = d.reshape(d.shape[0], self.heads, 128).norm(dim=2)
            bar = SIGMA_BAR * sig + (coh if coh is not None else 0.0)
            s = torch.where((n == 0) | (fr > DIFFUSE), torch.zeros_like(n), n / bar)
            i = int(s.argmax())
            out[name] = (e, float(s.reshape(-1)[i]), divmod(i, self.heads))
        return out

    def check(self, dq=None, dk=None, dv=None, label="", stat=True):
        """Both checks of each gradient given (the element bound only when stat is False); returns ratios() (every
        ratio checked must be <= 1)."""
        r = self.ratios(dq, dk, dv)
        for name, g in (("dq", dq), ("dk", dk), ("dv", dv)):
            if g is None:
                continue
            assert torch.isfinite(g.float()).all(), f"{label} {name}: non-finite gradient"
            e, s, (row, h) = r[name]
            print(f"attn_bwd_ref64 {label} {name}: element/bound {e:.3g}, norm/bar {s:.3g}")
            assert e <= 1.0, f"{label} {name}: |g - g64| reaches {e:.3g} x the per-element bound"
            assert s <= 1.0 or not stat, f"{label} {name}: the error norm of row {row}, head {h} is {s:.3g} x its bar"
        return r


def rel_l2(g, ref) -> float:
    return float((g.double().to(ref.device) - ref).norm() / ref.norm())


def emulate(q, k, v, dout, heads, scale, o=None, lse=None):
    """The kernels' arithmetic in torch fp32 with their roundings: bf16 P and dS into fp32 products, Delta from the bf16
    O, P = 2^(fp32(s sl2 - lse)).  o (bf16) and lse (fp32 [heads, Lq]) default to a float64 forward rounded like the
    kernel's outputs.  Returns bf16 (dq, dk, dv).  Test infrastructure: no kernel ordering or ex2.approx."""
    sl2 = scale_log2(scale)
    f32 = torch.float32
    Lq = q.shape[0]
    dq, dk, dv = (torch.empty(t.shape, dtype=torch.bfloat16, device=t.device) for t in (q, k, v))
    for h in range(heads):
        hs = slice(h * 128, (h + 1) * 128)
        qh, kh, vh, doh = (t[:, hs].to(f32) for t in (q, k, v, dout))
        if lse is None:
            x64 = (q[:, hs].double() @ k[:, hs].double().T) * sl2
            lse_h = torch.logsumexp(x64 * LN2, 1) / LN2
            oh = (torch.softmax(x64 * LN2, 1) @ v[:, hs].double()).to(torch.bfloat16).to(f32)
            lse_h = lse_h.to(f32)
        else:
            lse_h = lse[h].to(f32)
            oh = o[:, hs].to(f32)
        s = qh @ kh.T
        P = torch.exp2((s.double() * sl2 - lse_h.double()[:, None]).to(f32))  # fma: one rounding
        delta = (doh * oh).sum(1)
        dS = P * (doh @ vh.T - delta[:, None])
        Pb, dSb = P.to(torch.bfloat16).to(f32), dS.to(torch.bfloat16).to(f32)
        dv[:, hs] = (Pb.T @ doh).to(torch.bfloat16)
        dk[:, hs] = ((dSb.T @ qh) * scale).to(torch.bfloat16)
        dq[:, hs] = ((dSb @ kh) * scale).to(torch.bfloat16)
    assert Lq == q.shape[0]
    return dq, dk, dv


def lse_reference(q, k, heads, scale, block=1024):
    """(lse64 [heads, Lq], bound [heads, Lq]) of the forward's log-sum-exp in log2 units: |lse - lse64| <= MARGIN dlse
    with dlse of the module docstring (score, exponent and ex2 errors weighted by the row's softmax, the fp32 sum l
    over n_kv tiles, the fp32 m + log2(l))."""
    sl2 = scale_log2(scale)
    Lq, Lk = q.shape[0], k.shape[0]
    n_kv = (Lk + TILE - 1) // TILE
    lse = torch.empty(heads, Lq, dtype=torch.float64, device=q.device)
    bound = torch.empty_like(lse)
    for h in range(heads):
        hs = slice(h * 128, (h + 1) * 128)
        kh = k[:, hs].double()
        for r0 in range(0, Lq, block):
            qb = q[r0:r0 + block, hs].double()
            x = (qb @ kh.T) * sl2
            mx = x.amax(1, keepdim=True)
            p = torch.exp2(x - mx)
            w = p / p.sum(1, keepdim=True)
            eta_f = (LN2 * (sl2 * S_REL * (qb.abs() @ kh.abs().T) + U * ((x - mx).abs() + GUARD_LAG))
                     + EX2_REL).clamp(max=1.0)
            row = (mx + torch.log2(p.sum(1, keepdim=True)))[:, 0]
            lse[h, r0:r0 + block] = row
            bound[h, r0:r0 + block] = MARGIN * (((w * eta_f).sum(1) + (ACC_PER_TILE * n_kv + ACC_C) * U) / LN2
                                                + EX2_REL * (row.abs() + 32.0))
    return lse, bound
