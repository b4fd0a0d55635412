"""The tokenizer wrapper mirror (gen3c_b200/pretrained_vae.py) against a golden minted from the reference's own
VideoJITTokenizer on a tiny TorchScript checkpoint (tests/golden/vae_wrapper.npz, oracle/make_golden.py::mint_tokenizer):
temporal chunking, batch splitting, latent mean / std, dtype round trips, frame-count helpers."""
import os

import numpy as np
import pytest
import torch

from oracle import cases, golden


@pytest.mark.parametrize("tag,bf16", [("f32", False), ("bf16", True)])
def test_video_jit_tokenizer_matches_reference(tmp_path, golden_dir, tag, bf16):
    from gen3c_b200.pretrained_vae import VideoJITTokenizer

    g = golden.load(golden_dir, "vae_wrapper")
    cases.write_tiny_tokenizer(str(tmp_path))
    tok = VideoJITTokenizer(name="tiny", latent_ch=16, is_bf16=bf16, spatial_compression_factor=8,
                            temporal_compression_factor=8, pixel_chunk_duration=17, max_enc_batch_size=1,
                            max_dec_batch_size=1)
    tok.load_weights(str(tmp_path))
    x = cases.tiny_tokenizer_video()
    z = tok.encode(x)
    y = tok.decode(z)
    assert z.dtype == x.dtype and y.dtype == x.dtype
    np.testing.assert_array_equal(z.numpy(), g[f"z_{tag}"])   # same ops in the same order: bit-exact
    np.testing.assert_array_equal(y.numpy(), g[f"y_{tag}"])
    assert [tok.get_latent_num_frames(1), tok.get_latent_num_frames(34), tok.get_pixel_num_frames(6),
            tok.latent_chunk_duration] == list(g["frames"])
    with pytest.raises(AssertionError):
        tok.encode(x[:, :, :20])            # not a multiple of the 17-frame chunk
    with pytest.raises(AssertionError):
        tok.get_latent_num_frames(20)


def test_synthetic_tokenizer_shapes():
    from gen3c_b200.pretrained_vae import SyntheticVideoTokenizer

    tok = SyntheticVideoTokenizer(pixel_chunk_duration=17)
    x = cases.tiny_tokenizer_video()
    z = tok.encode(x)
    assert z.shape == (1, 16, 6, 2, 4)
    y = tok.decode(z)
    assert y.shape == x.shape and float(y.abs().max()) <= 1.0
    # the first three latent channels are the pooled image: a constant video survives the round trip
    c = torch.full_like(x, 0.25)
    assert torch.allclose(tok.decode(tok.encode(c)), c, atol=1e-2)
