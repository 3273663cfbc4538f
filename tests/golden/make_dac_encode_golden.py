"""Generate dac_encode.npz by EXECUTING transformers' DacModel.encode on the CPU -- the stand-in for descript-audio-codec
(not installed), whose encoder and quantizer it restates (transformers/models/dac/modeling_dac.py:442-472, :281-343).

Tiny codec: tiny_dac_cfg() with encoder_hidden_size 8 and downsampling_ratios [2, 4, 8, 8] (hop 512); weights
make_dac_weights(cfg, seed=2) (codebooks, out_proj, decoder) + make_dac_encoder_weights(cfg, seed=5).  The model runs in
float64, so the latents and codes are the network's exact values to ~1e-15.  The waveform's length is not a multiple of the
hop: it is right zero-padded first, as DACModel.encode's model.preprocess does (dac_wrapper/modeling_dac.py:64).

Stored: waveform [B, 1, L], padded [B, 1, L'], latents [B, latent, T] (encoder output), codes [B, K, T], and margins [K, B, T]:
each codebook's fp64 cosine-similarity gap between the best and the second-best codebook row along the reference's path.

Usage:  python tests/golden/make_dac_encode_golden.py
"""
from __future__ import annotations
import math
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

ENCODER = dict(encoder_hidden_size=8, downsampling_ratios=[2, 4, 8, 8])
SAMPLES = 2 * 512 * 5 + 300      # not a multiple of the hop


def encode_cfg():
    from oracle.config import tiny_dac_cfg
    return tiny_dac_cfg(**ENCODER)


def weights(cfg):
    from oracle.weights import make_dac_weights
    from tests.dac_encode_oracle import make_dac_encoder_weights
    w = make_dac_weights(cfg, seed=2)
    w.update(make_dac_encoder_weights(cfg, seed=5))
    return w


def waveform(B=2):
    g = torch.Generator().manual_seed(11)
    t = torch.arange(SAMPLES, dtype=torch.float64) / 44100.0
    tone = torch.stack([0.4 * torch.sin(2 * math.pi * f * t) for f in (220.0, 330.0)])[:B]
    return (tone + 0.1 * torch.randn(B, SAMPLES, generator=g, dtype=torch.float64)).float()[:, None, :]


def main():
    from transformers.models.dac import DacConfig, DacModel
    cfg = encode_cfg()
    hc = DacConfig(decoder_hidden_size=cfg.decoder_hidden_size, n_codebooks=cfg.n_codebooks, codebook_size=cfg.codebook_size,
                   codebook_dim=cfg.codebook_dim, hidden_size=cfg.hidden_size, upsampling_ratios=cfg.upsampling_ratios,
                   sampling_rate=44100, **ENCODER)
    m = DacModel(hc).eval()
    w = weights(cfg)
    sd = m.state_dict()
    assert set(sd) == set(w), set(sd) ^ set(w)
    for k, v in w.items():
        assert sd[k].shape == v.shape, (k, sd[k].shape, v.shape)
    m.load_state_dict(w)
    m = m.double()
    x = waveform()
    hop = math.prod(ENCODER["downsampling_ratios"])
    padded = F.pad(x, (0, math.ceil(SAMPLES / hop) * hop - SAMPLES))
    with torch.no_grad():
        xd = padded.double()
        codes = m.encode(xd).audio_codes
        z = m.encoder(xd)
        residual, margins = z, []
        for i, qz in enumerate(m.quantizer.quantizers):
            z_e = qz.in_proj(residual)
            B, D, T = z_e.shape
            sims = F.normalize(z_e.permute(0, 2, 1).reshape(B * T, D)) @ F.normalize(qz.codebook.weight).t()
            top2 = sims.topk(2, dim=1).values
            margins.append((top2[:, 0] - top2[:, 1]).reshape(B, T))
            assert torch.equal(sims.argmax(1).reshape(B, T), codes[:, i])
            residual = residual - qz(residual)[0]
    np.savez_compressed(os.path.join(HERE, "dac_encode.npz"), waveform=x.numpy(), padded=padded.numpy(), latents=z.numpy(),
                        codes=codes.numpy(), margins=torch.stack(margins).numpy())
    print("dac_encode.npz", codes.shape, "min margin", float(torch.stack(margins).min()))


if __name__ == "__main__":
    main()
