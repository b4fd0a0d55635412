"""The context-parallel branch of the attention kernel on one GPU, through g3c_attn_fwd_gated: the KV visit order rotated
to start at chunk `first` (K rows and the V^T chunk coordinate), the flag poll with its system-scope acquire, the proxy
fence before the TMA reads data published by a copy, and the wait_ns counter.  The engine's peer-memory mode is the only
caller of this branch and needs two GPUs; here the flags and the chunk data are published by this process's own copies.

The kernel's arithmetic depends only on the sequence of KV tiles it visits, so a gated launch from chunk c must be
bitwise equal to the ungated kernel on K and V^T whose chunks were rotated by c.  Every flag is raised before or during
each launch, so no case can wait for ever."""
import math
import time

import pytest
import torch

from tests import attn_ref64

pytestmark = pytest.mark.gpu

LN2 = math.log(2.0)
SEQ = 5


def bf(*shape, seed, s=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * s).to(torch.bfloat16)


def chunked_vt(v, chunks):
    """[chunks, D, chunk_len]: V^T chunk by chunk, the layout the engine's K/V^T exchange fills"""
    Lk, D = v.shape
    return v.reshape(chunks, Lk // chunks, D).permute(0, 2, 1).contiguous()


def rotated(k, vt, c):
    """K and V^T with their chunks rotated to start at chunk c"""
    cl = vt.shape[2]
    return torch.cat([k[c * cl:], k[:c * cl]]), torch.cat([vt[c:], vt[:c]])


def launch_gated(o, q, k, vt, heads, first, flags, seq, wait_ns, scale):
    from gen3c_b200 import _lib

    Lq, D = q.shape
    lib = _lib.load()
    _lib.check(lib.g3c_attn_fwd_gated(_lib.ptr(q), _lib.ptr(k), _lib.ptr(vt), _lib.ptr(o), Lq, k.shape[0], heads, D, D,
                                      D, vt.shape[2], scale, _lib.ptr(flags), seq, first, _lib.ptr(wait_ns),
                                      _lib.stream_ptr()), "g3c_attn_fwd_gated")
    return o


def gated(q, k, vt, heads, first, flags, seq=SEQ, scale=128 ** -0.5):
    """(o, wait_ns) of one gated launch, synchronised"""
    o = torch.empty_like(q)
    wait = torch.zeros(1, dtype=torch.int64, device="cuda")
    launch_gated(o, q, k, vt, heads, first, flags, seq, wait, scale)
    torch.cuda.synchronize()
    return o, int(wait)


def ungated(q, k, vt, heads, scale=128 ** -0.5):
    from gen3c_b200 import ops

    return ops.attention(q, k, vt, heads, scale=scale, vt_chunk_len=vt.shape[2])


def operands(Lq, chunks, cl, heads, seed):
    D = heads * 128
    q, k, v = bf(Lq, D, seed=seed), bf(chunks * cl, D, seed=seed + 1), bf(chunks * cl, D, seed=seed + 2)
    return q, k, v, chunked_vt(v, chunks)


# 1, 3 or 7 tiles per chunk: chunk boundaries at even and odd positions of the two-stage K / V rings
@pytest.mark.parametrize("cl", [128, 384, 896])
@pytest.mark.parametrize("chunks", [2, 3, 4, 8])
def test_rotation_with_flags_raised(chunks, cl):
    """Flags at or above seq before the launch: every first chunk gives the ungated kernel on rotated chunks bit for bit,
    differs from the unrotated order when first != 0, passes the float64 checks, and never waits."""
    heads = 1 + (chunks + cl // 128) % 4
    Lq = 77 + 64 * chunks  # ragged: the last query tile is partial
    q, k, v, vt = operands(Lq, chunks, cl, heads, seed=100 * chunks + cl // 128)
    flags = (SEQ + torch.arange(chunks, device="cuda", dtype=torch.int32)).contiguous()
    ref = attn_ref64.Reference(q, k, v, heads, 128 ** -0.5)
    o0 = ungated(q, k, vt, heads)
    for first in range(chunks):
        o, wait = gated(q, k, vt, heads, first, flags)
        assert wait == 0, (first, wait)
        kr, vtr = rotated(k, vt, first)
        assert torch.equal(o, ungated(q, kr, vtr, heads)), first
        assert torch.equal(o, o0) == (first == 0), first
        ref.check(o, f"chunks={chunks} cl={cl} first={first}")


def test_flag_comparison_wraps():
    """The flag test is a serial-number comparison: with seq = 2^32 - 1, flags that wrapped to 0 and 1 are later."""
    q, k, v, vt = operands(200, 3, 256, 2, seed=7)
    flags = torch.tensor([0, 1, -1], device="cuda", dtype=torch.int32)  # -1 is 2^32 - 1 = seq
    o, wait = gated(q, k, vt, 2, 1, flags, seq=0xFFFFFFFF)
    assert wait == 0
    kr, vtr = rotated(k, vt, 1)
    assert torch.equal(o, ungated(q, kr, vtr, 2))


@pytest.mark.parametrize("cp", [2, 4])
def test_engine_call_shape(cp):
    """The p2p engine's self-attention launch at the benchmark's size: Lq = L = 56 320 / cp tokens of rank `rank`,
    Lk = 56 320 keys in cp chunks of L, 32 heads, Q in log2 units (scale ln 2), first = rank."""
    L_all, heads = 56320, 32
    L, D = L_all // cp, heads * 128
    q = (bf(L_all, D, seed=200) * (128 ** -0.5 * math.log2(math.e))).to(torch.bfloat16)
    k, v = bf(L_all, D, seed=201), bf(L_all, D, seed=202)
    vt = chunked_vt(v, cp)
    flags = torch.full((cp,), SEQ, device="cuda", dtype=torch.int32)
    gen = torch.Generator(device="cuda").manual_seed(203)
    for rank in range(cp):
        qr = q[rank * L:(rank + 1) * L]
        o, wait = gated(qr, k, vt, heads, rank, flags, scale=LN2)
        assert wait == 0
        kr, vtr = rotated(k, vt, rank)
        assert torch.equal(o, ungated(qr, kr, vtr, heads, scale=LN2)), rank
        del kr, vtr
        rows = torch.randint(0, L, (64,), device="cuda", generator=gen)
        attn_ref64.check(o, qr, k, v, heads, LN2, rows=rows, label=f"cp={cp} rank={rank}")


@pytest.mark.parametrize("chunks,cl,first,Lq,heads", [(4, 384, 1, 300, 2), (2, 896, 1, 2048, 12), (8, 128, 5, 130, 1)])
def test_late_publication(chunks, cl, first, Lq, heads):
    """The p2p exchange in one process: the remote chunks of K and V^T hold NaN and every flag (remote, local and two
    spare slots) sits at seq - 1 when the kernel is launched on stream A.  0.5 s later stream B copies the real chunk
    data from pinned host memory, then all flags at seq (the engine's order: data, then a 4-byte flag copy on the same
    stream).  The output must be bitwise that of the launch with every flag raised in advance, and the loader must have
    waited.  (Heads x query tiles = 192 CTAs in the second case: more than fit at once, so some start after the
    publication.)"""
    q, k, v, vt = operands(Lq, chunks, cl, heads, seed=300 + chunks)
    want, _ = gated(q, k, vt, heads, first, torch.full((chunks,), SEQ, device="cuda", dtype=torch.int32))
    k_host, vt_host = k.cpu().pin_memory(), vt.cpu().pin_memory()
    flags_host = torch.full((chunks + 2,), SEQ, dtype=torch.int32).pin_memory()
    k_late, vt_late = k.clone(), vt.clone()
    remote = [c for c in range(chunks) if c != first]
    for c in remote:
        k_late[c * cl:(c + 1) * cl] = float("nan")
        vt_late[c] = float("nan")
    flags = torch.full((chunks + 2,), SEQ - 1, device="cuda", dtype=torch.int32)
    wait = torch.zeros(1, dtype=torch.int64, device="cuda")
    o = torch.empty_like(q)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(sa):
        launch_gated(o, q, k_late, vt_late, heads, first, flags, SEQ, wait, 128 ** -0.5)
    time.sleep(0.5)
    with torch.cuda.stream(sb):
        for c in remote:
            k_late[c * cl:(c + 1) * cl].copy_(k_host[c * cl:(c + 1) * cl], non_blocking=True)
            vt_late[c].copy_(vt_host[c], non_blocking=True)
        flags.copy_(flags_host, non_blocking=True)
    torch.cuda.synchronize()
    assert int(wait) > 0
    assert torch.equal(o, want)
