"""CPU restatement of DACModel.encode (test infrastructure only).

DACModel.encode (dac_wrapper/modeling_dac.py:33-104) = model.preprocess (right zero-pad to the hop, :64) + model.encode (:95).
descript-audio-codec is not installed; the arithmetic is restated from transformers' DacModel, which restates the same network:
  encoder                       transformers/models/dac/modeling_dac.py:442-472   block :210-231   residual unit :173-207
  residual vector quantizer     :281-343   vector quantize :102-170
Built on oracle/dac.py's OracleDAC (snake, the residual unit); tests/golden/dac_encode.npz, written by transformers'
DacModel.encode, pins it.  Encoder shape keys follow transformers' DacConfig: encoder_hidden_size (default 64) and
downsampling_ratios (default [2, 4, 8, 8]).
"""
from __future__ import annotations
import math

import torch
import torch.nn.functional as F

from oracle.config import Cfg
from oracle.dac import OracleDAC, snake


class OracleDACEncoder(OracleDAC):
    def encoder_rates(self):
        return list(self.cfg.get("downsampling_ratios", [2, 4, 8, 8]))

    def encoder(self, x: torch.Tensor) -> torch.Tensor:
        """Padded waveform [B, 1, L] -> latents [B, latent, L / hop]."""
        w = self.w
        x = F.conv1d(x, w["encoder.conv1.weight"], w["encoder.conv1.bias"], padding=3)
        for bi, s in enumerate(self.encoder_rates()):
            p = f"encoder.block.{bi}."
            for ri, dil in ((1, 1), (2, 3), (3, 9)):
                x = self._res(x, p + f"res_unit{ri}.", dil)
            x = snake(x, w[p + "snake1.alpha"])
            x = F.conv1d(x, w[p + "conv1.weight"], w[p + "conv1.bias"], stride=s, padding=math.ceil(s / 2))
        x = snake(x, w["encoder.snake1.alpha"])
        return F.conv1d(x, w["encoder.conv2.weight"], w["encoder.conv2.bias"], padding=1)

    def quantize(self, z: torch.Tensor, n_q: int | None = None, follow: torch.Tensor | None = None):
        """latents [B, latent, T] -> (codes [B, n_q, T], per-codebook cosine similarities [B, T, codebook_size]).

        follow [B, >= n_q, T]: take these codes instead of the argmax for the residual update (to re-trace another
        implementation's path and see how close each of its choices was)."""
        w = self.w
        residual = z
        codes, sims = [], []
        for i in range(n_q or self.cfg.n_codebooks):
            q = f"quantizer.quantizers.{i}."
            z_e = F.conv1d(residual, w[q + "in_proj.weight"], w[q + "in_proj.bias"])
            B, D, T = z_e.shape
            enc = F.normalize(z_e.permute(0, 2, 1).reshape(B * T, D))
            cb = F.normalize(w[q + "codebook.weight"])
            dist = -(enc.pow(2).sum(1, keepdim=True) - 2 * enc @ cb.t()) + cb.pow(2).sum(1, keepdim=True).t()
            idx = dist.max(1)[1].reshape(B, T) if follow is None else follow[:, i].to(torch.int64)
            sims.append((enc @ cb.t()).reshape(B, T, -1))
            z_q = F.embedding(idx, w[q + "codebook.weight"]).transpose(1, 2)
            z_q = z_e + (z_q - z_e)   # straight-through: the forward value of z_e + (z_q - z_e).detach()
            residual = residual - F.conv1d(z_q, w[q + "out_proj.weight"], w[q + "out_proj.bias"])
            codes.append(idx)
        return torch.stack(codes, dim=1), sims

    def encode(self, input_values: torch.Tensor, n_q: int | None = None) -> torch.Tensor:
        """DACModel.encode: input_values [B, 1, L] -> audio_codes [1, B, n_q, ceil(L / hop)]."""
        hop = math.prod(self.encoder_rates())
        length = input_values.shape[-1]
        right_pad = math.ceil(length / hop) * hop - length   # model.preprocess
        x = F.pad(input_values.to(self.dtype), (0, right_pad))
        codes, _ = self.quantize(self.encoder(x), n_q)
        return codes[None]


def make_dac_encoder_weights(cfg: Cfg, seed: int = 0) -> dict[str, torch.Tensor]:
    """Folded DAC encoder + quantizer in_proj weights, fp32 (the codebooks and out_proj come from oracle.weights.make_dac_weights).

    Keys follow transformers.models.dac.DacModel: encoder.conv1, encoder.block.N.{res_unitM.{snake1,conv1,snake2,conv2},
    snake1.alpha,conv1}, encoder.snake1.alpha, encoder.conv2, quantizer.quantizers.N.in_proj.  A generator of its own, fan-in
    scales so activations stay O(1) through the stack."""
    g = torch.Generator().manual_seed(seed)

    def conv(co, ci, k):
        s = 1.0 / math.sqrt(ci * k)
        return torch.randn(co, ci, k, generator=g) * s, torch.randn(co, generator=g) * 0.02

    def alpha(c):
        return (1.0 + 0.3 * torch.randn(1, c, 1, generator=g)).abs() + 0.1

    d = cfg.get("encoder_hidden_size", 64)
    w: dict[str, torch.Tensor] = {}
    w["encoder.conv1.weight"], w["encoder.conv1.bias"] = conv(d, 1, 7)
    for bi, s in enumerate(cfg.get("downsampling_ratios", [2, 4, 8, 8])):
        p = f"encoder.block.{bi}."
        for ri in (1, 2, 3):
            r = p + f"res_unit{ri}."
            w[r + "snake1.alpha"] = alpha(d)
            ww, bb = conv(d, d, 7)
            w[r + "conv1.weight"], w[r + "conv1.bias"] = ww * 0.5, bb
            w[r + "snake2.alpha"] = alpha(d)
            ww, bb = conv(d, d, 1)
            w[r + "conv2.weight"], w[r + "conv2.bias"] = ww * 0.5, bb
        w[p + "snake1.alpha"] = alpha(d)
        w[p + "conv1.weight"], w[p + "conv1.bias"] = conv(2 * d, d, 2 * s)
        d *= 2
    w["encoder.snake1.alpha"] = alpha(d)
    w["encoder.conv2.weight"], w["encoder.conv2.bias"] = conv(cfg.hidden_size, d, 3)
    for i in range(cfg.n_codebooks):
        w[f"quantizer.quantizers.{i}.in_proj.weight"], w[f"quantizer.quantizers.{i}.in_proj.bias"] = conv(cfg.codebook_dim, cfg.hidden_size, 1)
    return w
