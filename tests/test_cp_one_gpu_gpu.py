"""The engine's context- and CFG-parallel exchanges run on one GPU: one handle per rank in this process, their regions
wired together with g3c_dit_cp_attach / g3c_dit_cfg_attach instead of IPC, the ranks run one after another.

A rank never waits.  Before it is launched, every flag it can read is at the seq it compares against: the ranks that
ran earlier raised theirs with their own pushes (their chunks are the engine's real output), and the test publishes
the rest, with the replay's chunks for the ranks that have not run yet.  Each launch is preceded by a read-back of the
rank's flags that asserts this, so a push that left a flag low fails an assert and never spins a kernel.  Two layer-
parity sets hold every chunk of a forward only for nets of at most two blocks; larger nets need concurrent ranks.

Each rank's output is torch.equal to the multi-rank operator replay of tests/engine_replay.py, and the ranks together
stay near the single-handle forward over all frames, where replays with the remote chunks dropped, with every rank on
the first frame's tables or with the other parity set miss by 3x.  The nets carry signal through their attention
(tests/test_engine_signal_gpu.py): with the weights of random_state_dict those broken forwards would pass a rel-L2 bar.
"""
import ctypes as C
import dataclasses
import math

import pytest
import torch

from gen3c_b200 import _lib, sampler
from oracle import cases, dit_oracle
from tests import engine_replay as er
from tests.test_engine_signal_gpu import build_net, rel, signal_state_dict

pytestmark = pytest.mark.gpu

bf = torch.bfloat16
EINVAL, ESTATE = -1, -4
M = 128  # context tokens
# latent (T_local, H, W) of one rank: T_local * Hp * Wp = 128 tokens, one KV tile per chunk
GRIDS = {"square": (2, 16, 16), "nonsquare": (1, 16, 32)}
# (rel-L2, largest element difference / largest element) of the ranks together against the single-handle forward over
# all frames, per Linear mode.  Ranks > 0 visit the KV chunks in a rotated order, which changes the roundings of their
# attention sums.  On an H100 80GB HBM3 (700 W) the 16 cases reach 2.6e-3 / 6.7e-3 in bf16 and 7.2e-3 / 1.6e-2 in fp8, where the per-row e4m3
# quantisation of the activations magnifies a changed bf16 rounding; the broken replays are at least 9.8e-2 / 1.3e-1.
BARS = {False: (4e-3, 1e-2), True: (1e-2, 2.5e-2)}


def tiny(blocks):
    return dataclasses.replace(cases.TINY, num_blocks=blocks)


def device_bytes(ptr, nbytes):
    """A uint8 tensor over device memory the engine owns (no copy; valid while the handle keeps it)."""

    class Mem:
        __cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}

    return torch.as_tensor(Mem(), device="cuda")


class CpRegion:
    """One rank's context-parallel region as views: k[s] [cp, L, D] and vt[s] [cp, D, L] bf16 of parity set s, and
    flags [16] (int32; slot s*8 + r = seq of the last layer whose rank-r chunk landed in set s)."""

    def __init__(self, net, cp, L, D):
        base, ok, ov, of = C.c_void_p(), (C.c_int64 * 2)(), (C.c_int64 * 2)(), C.c_int64()
        _lib.check(_lib.load().g3c_dit_cp_region(net._engine(), C.byref(base), ok, ov, C.byref(of)), "g3c_dit_cp_region")
        self.base = base.value
        chunk = cp * L * D * 2
        view = lambda off: device_bytes(self.base + off, chunk).view(bf)  # noqa: E731
        self.k = [view(ok[s]).view(cp, L, D) for s in (0, 1)]
        self.vt = [view(ov[s]).view(cp, D, L) for s in (0, 1)]
        self.flags = device_bytes(self.base + of.value, 64).view(torch.int32)


def cp_ranks(cfg, sd, fp8, cp, T, H, W):
    """One engine handle per rank in peer-memory context-parallel mode, shaped and attached to each other."""
    nets = []
    for r in range(cp):
        net = build_net(cfg, sd, fp8)
        _lib.check(_lib.load().g3c_dit_enable_cp(net._engine(), None, r, cp), "g3c_dit_enable_cp")
        net._sync_weights()
        net._set_shape(T, H, W, M, 24.0)
        nets.append(net)
    L = T * (H // 2) * (W // 2)
    regions = [CpRegion(n, cp, L, cfg.model_channels) for n in nets]
    bases = (C.c_void_p * cp)(*[rg.base for rg in regions])
    for n in nets:
        _lib.check(_lib.load().g3c_dit_cp_attach(n._engine(), bases, cp), "g3c_dit_cp_attach")
    return nets, regions


def signal_inputs(cfg, T, H, W, seed):
    inp = cases.dit_inputs(cfg, T=T, H=H, W=W, ctx_len=M, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    inp["padding"] = (torch.rand(H, W, generator=g) < 0.3).float()
    d = lambda t: t.to(bf).cuda().contiguous()  # noqa: E731
    return {k: d(v) if torch.is_tensor(v) else v for k, v in inp.items()}


def elem(a, b):
    """largest element difference relative to the largest element of b"""
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("grid", list(GRIDS))
@pytest.mark.parametrize("cp", [2, 4])
@pytest.mark.parametrize("blocks", [1, 2])
@torch.no_grad()
def test_cp_ranks_equal_replay(blocks, cp, grid, fp8):
    """Two forwards per rank handle (cond with pose, then uncond without, one timestep), so that the second one's
    layers reuse the parity sets with seqs blocks+1 .. 2*blocks.  Per rank: launches per category, no flag wait, output
    torch.equal to the replay; after it, every peer region holds its K and V^T chunk of every layer, torch.equal to the
    replay, in the layer's set, with the flag at the layer's seq.  The ranks concatenated are within BARS of the
    single-handle forward over all frames; replay variants miss both bars by 3x."""
    cfg = tiny(blocks)
    T, H, W = GRIDS[grid]
    L = T * (H // 2) * (W // 2)
    sd = signal_state_dict(cfg, seed=0)
    inp = signal_inputs(cfg, cp * T, H, W, seed=1)
    ts = inp["timestep"]

    full = build_net(cfg, sd, fp8)  # the unsharded forward
    full._sync_weights()
    full._set_shape(cp * T, H, W, M, 24.0)
    mods, modf = er.read_modulation(full, ts)  # the adaLN vectors depend on the weights and the timestep only
    nets, regions = cp_ranks(cfg, sd, fp8, cp, T, H, W)
    tables = [er.read_tables(n, r * T, L) for r, n in enumerate(nets)]
    wsd = {k: v for k, v in nets[0].state_dict().items() if k != "pos_embedder.seq"}
    sl = lambda t, r: None if t is None else t[:, r * T:(r + 1) * T].contiguous()  # noqa: E731

    for rnd, (pose, ctx) in enumerate(((inp["pose"], inp["ctx_c"]), (None, inp["ctx_u"]))):
        ranks = [(sl(inp["x"], r), sl(inp["cond_mask"], r), sl(pose, r), inp["padding"], *tables[r]) for r in range(cp)]
        want, kv = er.replay(wsd, cfg, ranks, ctx, mods, modf, fp8)
        seqs = [rnd * blocks + i + 1 for i in range(blocks)]  # kv_seq of each self-attention layer of this round
        outs = []
        for r, net in enumerate(nets):
            own = regions[r]
            # all published: the earlier ranks' pushes raised their flags; the test publishes the later ranks' chunks
            # (none for the last rank) and every other slot of the layer's set, this rank's own included
            torch.cuda.synchronize()
            flags = own.flags.cpu()
            for i, s in enumerate(seqs):
                st = s & 1
                for c in range(r):
                    assert int(flags[st * 8 + c]) == s, (f"round {rnd} rank {r}: the flag of rank {c}'s layer {i} push "
                                                         f"is {int(flags[st * 8 + c])}, not {s}")
                for c in range(r + 1, cp):
                    own.k[st][c].copy_(kv[i][0][c * L:(c + 1) * L])
                    own.vt[st][c].copy_(kv[i][1][c])
                own.flags[st * 8 + r:st * 8 + 8] = s
            torch.cuda.synchronize()
            flags = own.flags.cpu()
            assert all(int(flags[(s & 1) * 8 + c]) == s for s in seqs for c in range(8)), flags

            out, n, wait = er.engine_forward(net, *ranks[r][:4], ts, ctx)
            assert n == er.launches(blocks, fp8, vectors=rnd == 0), (r, n)
            assert wait == 0.0, (r, wait)
            assert torch.equal(out, want[r]), (rnd, r, float((out.float() - want[r].float()).abs().max()))
            outs.append(out)
            for p in range(cp):
                if p == r:
                    continue
                for i, s in enumerate(seqs):
                    st = s & 1
                    assert torch.equal(regions[p].k[st][r], kv[i][0][r * L:(r + 1) * L]), (rnd, r, p, i)
                    assert torch.equal(regions[p].vt[st][r], kv[i][1][r]), (rnd, r, p, i)
                    assert int(regions[p].flags[st * 8 + r]) == s, (rnd, r, p, i)
            # retire what the test published: the later ranks' pushes must write these chunks and flags themselves
            for s in seqs:
                own.k[s & 1][r + 1:] = float("nan")
                own.vt[s & 1][r + 1:] = float("nan")
                own.flags[(s & 1) * 8 + r + 1:(s & 1) * 8 + cp] = 0

        got = torch.cat(outs, dim=1)
        ref, _, _ = er.engine_forward(full, inp["x"], inp["cond_mask"], pose, inp["padding"], ts, ctx)
        errs = {"ranks": (rel(got, ref), elem(got, ref))}
        if rnd == 0:
            other = lambda i, k, vt: kv[i ^ 1] if blocks == 2 else (torch.zeros_like(k), torch.zeros_like(vt))  # noqa: E731
            variants = {
                "remote_dropped": er.replay(wsd, cfg, ranks, ctx, mods, modf, fp8, drop_remote=True)[0],
                "tables_t0": er.replay(wsd, cfg, [(*rk[:4], *tables[0]) for rk in ranks], ctx, mods, modf, fp8)[0],
                # the other set holds the other block's chunks, or nothing yet in a one-block net's first forward
                "other_set": er.replay(wsd, cfg, ranks, ctx, mods, modf, fp8, self_kv=other)[0],
            }
            for name, outs_v in variants.items():
                b = torch.cat(outs_v, dim=1)
                errs[name] = (rel(b, ref), elem(b, ref))
        print(f"blocks {blocks} cp {cp} {grid} {'fp8' if fp8 else 'bf16'} round {rnd}, rel-L2 / element vs the "
              "unsharded forward: " + ", ".join(f"{k} {a:.2e} / {b:.2e}" for k, (a, b) in errs.items()))
        bar_rel, bar_elem = BARS[fp8]
        assert errs["ranks"][0] <= bar_rel and errs["ranks"][1] <= bar_elem, errs
        for name, (a, b) in errs.items():
            assert name == "ranks" or (a >= 3 * bar_rel and b >= 3 * bar_elem), (name, errs)


class CfgRegion:
    """One role's CFG exchange region as views: slot[i] bf16 [16, T, H, W] (the partner's output of step seq in slot
    seq & 1) and flags [2] int32."""

    def __init__(self, net, T, H, W):
        base, slot_bytes = C.c_void_p(), C.c_int64()
        _lib.check(_lib.load().g3c_dit_cfg_region(net._engine(), C.byref(base), C.byref(slot_bytes)),
                   "g3c_dit_cfg_region")
        self.base, n = base.value, 16 * T * H * W
        self.slot = [device_bytes(self.base + i * slot_bytes.value, 2 * n).view(bf).view(16, T, H, W) for i in (0, 1)]
        self.flags = device_bytes(self.base + 2 * slot_bytes.value, 8).view(torch.int32)


def read_step(net, like):
    """x~, x_in, cond and uncond network outputs of the last g3c_denoise_step"""
    bufs = [torch.empty_like(like) for _ in range(4)]
    _lib.check(_lib.load().g3c_dit_read_step(net._engine(), *(b.data_ptr() for b in bufs), _lib.stream_ptr()),
               "g3c_dit_read_step")
    torch.cuda.synchronize()
    return bufs


@torch.no_grad()
def test_cfg_parallel_step_equals_unsharded():
    """Two g3c_denoise_step calls of a CFG pair (role 0 cond, role 1 uncond) attached in-process, so both exchange slots
    are used.  Role 0 runs first on role 1's branch output published by the test, role 1 then on what role 0 pushed.
    x_next, the CFG-combined network output and g3c_dit_read_step of both roles are torch.equal to the unsharded step;
    each push lands in the partner's slot seq & 1 with the flag at seq."""
    cfg = tiny(2)
    T, H, W = 2, 16, 16
    sd = signal_state_dict(cfg, seed=3)
    inp = signal_inputs(cfg, T, H, W, seed=4)
    sig = dit_oracle.karras_sigmas(35)
    noise = torch.from_numpy(dit_oracle.arch_invariant_rand((16, T, H, W), 1)).cuda()
    ind = torch.zeros(T, device="cuda")
    ind[0] = 1.0
    x0 = (inp["x"].float() * math.sqrt(float(sig[20]) ** 2 + 0.25)).to(bf)

    def step(net, xt, k):
        o = torch.empty_like(xt)
        x = sampler.denoise_step(net, xt, inp["gt"], noise, ind, inp["cond_mask"], inp["pose"], inp["padding"],
                                 inp["ctx_c"], inp["ctx_u"], float(sig[20 + k]), float(sig[21 + k]), 1.5,
                                 net_output=o)
        torch.cuda.synchronize()
        return x, o

    full = build_net(cfg, sd)
    want = []
    xt = x0
    for k in range(2):
        x, o = step(full, xt, k)
        want.append((x, o, read_step(full, x)))
        xt = x
    assert not torch.equal(want[0][2][2], want[0][2][3])

    roles = []
    for role in (0, 1):
        net = build_net(cfg, sd)
        _lib.check(_lib.load().g3c_dit_enable_cfg_parallel(net._engine(), role), "g3c_dit_enable_cfg_parallel")
        net._sync_weights()
        net._set_shape(T, H, W, M, 24.0)
        roles.append(net)
    reg = [CfgRegion(n, T, H, W) for n in roles]
    for role in (0, 1):
        _lib.check(_lib.load().g3c_dit_cfg_attach(roles[role]._engine(), reg[1 - role].base), "g3c_dit_cfg_attach")

    xt = x0
    for k in range(2):
        s = k + 1  # cfg_seq: reset by set_shape, one per step
        slot = s & 1
        w_x, w_o, (w_xt, w_xin, w_oc, w_ou) = want[k]
        # role 0: the test publishes role 1's branch output; both flags at seq, so a wrong slot cannot wait
        reg[0].slot[slot].copy_(w_ou)
        reg[0].flags[:] = s
        torch.cuda.synchronize()
        x, o = step(roles[0], xt, k)
        assert torch.equal(x, w_x) and torch.equal(o, w_o), k
        assert int(reg[1].flags[slot]) == s and torch.equal(reg[1].slot[slot], w_oc), k
        reg[0].slot[slot].fill_(float("nan"))  # retired: role 1's push must write it again
        reg[0].flags[slot] = 0
        # role 1 runs on what role 0 pushed; the other slot's flag, which no push raises, is published
        torch.cuda.synchronize()
        assert int(reg[1].flags[slot]) == s
        reg[1].flags[1 - slot] = s
        x, o = step(roles[1], xt, k)
        assert torch.equal(x, w_x) and torch.equal(o, w_o), k
        assert int(reg[0].flags[slot]) == s and torch.equal(reg[0].slot[slot], w_ou), k
        for net in roles:
            for got, ref in zip(read_step(net, x), (w_xt, w_xin, w_oc, w_ou)):
                assert torch.equal(got, ref), k
        xt = x


@torch.no_grad()
def test_attach_errors():
    """Region queries without a region are G3C_ESTATE; attach before set_shape is G3C_ESTATE, with a wrong count, a null
    entry or a foreign own entry G3C_EINVAL.  None of them writes to a region, and a correct attach succeeds after."""
    lib = _lib.load()
    cfg = tiny(1)
    sd = dit_oracle.random_state_dict(cfg, seed=0)
    base, ok, ov, of, sb = C.c_void_p(), (C.c_int64 * 2)(), (C.c_int64 * 2)(), C.c_int64(), C.c_int64()

    plain = build_net(cfg, sd)
    plain._sync_weights()
    plain._set_shape(2, 16, 16, M, 24.0)
    assert lib.g3c_dit_cp_region(plain._engine(), C.byref(base), ok, ov, C.byref(of)) == ESTATE
    assert lib.g3c_dit_cfg_region(plain._engine(), C.byref(base), C.byref(sb)) == ESTATE

    nets = [build_net(cfg, sd) for _ in range(2)]
    for r, n in enumerate(nets):
        _lib.check(lib.g3c_dit_enable_cp(n._engine(), None, r, 2), "g3c_dit_enable_cp")
    h0 = nets[0]._engine()
    assert lib.g3c_dit_cp_region(h0, C.byref(base), ok, ov, C.byref(of)) == ESTATE
    assert lib.g3c_dit_cp_attach(h0, (C.c_void_p * 2)(1024, 2048), 2) == ESTATE
    for n in nets:
        n._sync_weights()
        n._set_shape(2, 16, 16, M, 24.0)
    regions = [CpRegion(n, 2, 128, cfg.model_channels) for n in nets]
    b0, b1 = regions[0].base, regions[1].base
    assert lib.g3c_dit_cp_attach(h0, (C.c_void_p * 1)(b0), 1) == EINVAL
    assert lib.g3c_dit_cp_attach(h0, (C.c_void_p * 3)(b0, b1, b1), 3) == EINVAL
    assert lib.g3c_dit_cp_attach(h0, (C.c_void_p * 2)(b0, None), 2) == EINVAL
    assert lib.g3c_dit_cp_attach(h0, (C.c_void_p * 2)(b1, b0), 2) == EINVAL
    assert lib.g3c_dit_cp_attach(h0, None, 2) == EINVAL
    torch.cuda.synchronize()
    for rg in regions:
        assert not rg.flags.any() and not rg.k[0].any() and not rg.vt[1].any()
    assert lib.g3c_dit_cp_attach(h0, (C.c_void_p * 2)(b0, b1), 2) == 0

    cfgp = build_net(cfg, sd)
    _lib.check(lib.g3c_dit_enable_cfg_parallel(cfgp._engine(), 0), "g3c_dit_enable_cfg_parallel")
    assert lib.g3c_dit_cfg_region(cfgp._engine(), C.byref(base), C.byref(sb)) == ESTATE
    assert lib.g3c_dit_cfg_attach(cfgp._engine(), b1) == ESTATE
    cfgp._sync_weights()
    cfgp._set_shape(2, 16, 16, M, 24.0)
    assert lib.g3c_dit_cfg_attach(cfgp._engine(), None) == EINVAL
    rg = CfgRegion(cfgp, 2, 16, 16)
    assert not rg.flags.any() and not rg.slot[1].any()
    assert lib.g3c_dit_cfg_attach(cfgp._engine(), b1) == 0


@pytest.mark.parametrize("first", [0, 1])
@torch.no_grad()
def test_destroy_attached_handles(first):
    """Handles whose regions are attached to each other (context- and CFG-parallel) are destroyed in either order: the
    engine frees its own regions and unmaps no attached pointer, so no CUDA error is left behind and the survivor's
    region stays readable."""
    lib = _lib.load()
    cfg = tiny(1)
    sd = dit_oracle.random_state_dict(cfg, seed=0)
    nets = []
    for r in range(2):
        net = build_net(cfg, sd)
        _lib.check(lib.g3c_dit_enable_cp(net._engine(), None, r, 2), "g3c_dit_enable_cp")
        _lib.check(lib.g3c_dit_enable_cfg_parallel(net._engine(), r), "g3c_dit_enable_cfg_parallel")
        net._sync_weights()
        net._set_shape(2, 16, 16, M, 24.0)
        nets.append(net)
    regions = [CpRegion(n, 2, 128, cfg.model_channels) for n in nets]
    bases = (C.c_void_p * 2)(*[rg.base for rg in regions])
    cfg_reg = [CfgRegion(n, 2, 16, 16) for n in nets]
    for r, n in enumerate(nets):
        _lib.check(lib.g3c_dit_cp_attach(n._engine(), bases, 2), "g3c_dit_cp_attach")
        _lib.check(lib.g3c_dit_cfg_attach(n._engine(), cfg_reg[1 - r].base), "g3c_dit_cfg_attach")
    survivor = 1 - first
    regions[survivor].flags[:] = 7
    cfg_reg[survivor].flags[:] = 9
    for net in (nets[first], nets[survivor]):
        _lib.check(lib.g3c_dit_destroy(net._handle), "g3c_dit_destroy")
        net._handle = None
        torch.cuda.synchronize()
        assert float(torch.ones(256, device="cuda").sum()) == 256.0  # no CUDA error is pending
        if net is nets[first]:
            assert int(regions[survivor].flags.sum()) == 7 * 16 and int(cfg_reg[survivor].flags.sum()) == 18
