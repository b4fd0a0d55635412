"""Parity of the DiT engine at the BASELINE configuration (SURVEY.md §8c; VERDICT r01 item 1), all through the C ABI.

(a) ONE block at the full 7B width (D=4096, 32 heads, ffn 16 384, ctx 512x1024, the real position tables) on two latent
    frames of the 720p grid (7 040 tokens) against the golden minted from the REFERENCE'S OWN class in fp32
    (tests/golden/dit_fullwidth.npz, oracle/make_golden.py::mint_dit_fullwidth).
(b) the 28-block 7B network at 7 040 tokens and (c) at the full 56 320 tokens against the fp32 oracle graph run on the
    GPU (oracle/parity.py; the restated oracle equals the reference's class to rel-L2 0 on (a)).

Tolerance.  north_star asks for 1e-3 relative.  The reference itself computes in bf16: the same graph with every tensor
stored in bf16 sits at 7e-3 (one block) ... 3e-2 (28 blocks) from its own fp32 result, so 1e-3 against fp32 is not
reachable by any bf16-operand implementation, the reference included.  The bar asserted here is therefore
    err(engine vs fp32) <= err(bf16 run of the reference graph vs fp32)    at every depth,
i.e. the engine is at least as close to the exact result as the reference's own precision, plus an absolute cap that
catches gross errors."""
import os

import numpy as np
import pytest
import torch

from oracle import cases, dit_oracle, golden, parity

pytestmark = pytest.mark.gpu


def test_fullwidth_block_matches_reference_golden(golden_dir):
    g = golden.load(golden_dir, "dit_fullwidth")
    cfg, shp = cases.FULLWIDTH_1BLOCK, cases.FULLWIDTH_SHAPE
    sd = dit_oracle.random_state_dict(cfg, seed=21)      # the CPU generator: same numbers as when the golden was minted
    net = parity.build_engine_net(cfg, sd, 1, "cuda")
    inp = cases.dit_inputs(cfg, **shp, seed=22)
    got = parity.engine_forward(net, inp, shp["T"], torch.device("cuda")).cpu()
    err = parity.rel_l2(got, torch.from_numpy(g["out_cond"]))
    floor = float(g["oracle_bf16_rel_l2"])
    print(f"full-width block: engine vs reference fp32 golden rel-L2 {err:.3e} (bf16 run of the same graph: {floor:.3e})")
    assert err < 5e-3 and err < floor


def test_7b_28_blocks_7040_tokens_matches_fp32_oracle():
    res = parity.depth_sweep(T=2, depths=(2, 28))
    for nb, r in res.items():
        assert r["engine"] <= r["bf16"], (nb, r)
    assert res[2]["engine"] < 5e-3 and res[28]["engine"] < 3e-2, res


@pytest.mark.timeout(900)
def test_7b_28_blocks_full_56320_tokens_matches_fp32_oracle():
    """The BASELINE workload itself: latent [16,16,88,160], 28 blocks; the engine takes the same GEMM and attention
    paths as bench.py.  The fp32 oracle costs ~2.2e15 fp32 FLOP on the GPU."""
    res = parity.depth_sweep(T=16, depths=(28,), with_bf16=False)
    assert res[28]["engine"] < 3e-2, res
