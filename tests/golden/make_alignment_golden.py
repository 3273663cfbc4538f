"""Writes tests/golden/alignment.npz: transformers' Whisper token-timestamp steps on alignment matrices.

For each case, x [F, P] (frames x transcript tokens, fp32) goes through transformers.models.whisper.generation_whisper
._median_filter(width 7) along frames and _dynamic_time_warping(-filtered) as WhisperForConditionalGeneration
._extract_token_timestamps runs them; the fixture keeps x, the filtered matrix and the jump frames (the first frame of each
token on the path).  Cases: random, coarsely quantized (many tied costs), constant (every cost tied), monotone diagonal bands,
more tokens than frames, and 1 to 4 frames (the filter's pass-through edge).

Run: python tests/golden/make_alignment_golden.py  (needs transformers; the tests only read the .npz)
"""
import os

import numpy as np
import torch
from transformers.models.whisper.generation_whisper import _dynamic_time_warping, _median_filter

WIDTH = 7


def cases():
    g = np.random.default_rng(1234)
    out = {}
    for i, (F, P) in enumerate([(40, 7), (97, 13), (300, 32), (5, 9)]):
        out[f"random{i}"] = g.random((F, P), dtype=np.float32)
    for i, (F, P) in enumerate([(33, 6), (64, 16)]):
        out[f"tied{i}"] = (g.integers(0, 4, size=(F, P)) / 4).astype(np.float32)
    out["constant"] = np.full((21, 5), 0.25, dtype=np.float32)
    for i, (F, P) in enumerate([(120, 10), (50, 50)]):
        f = np.arange(F)[:, None] / F
        p = np.arange(P)[None, :] / P
        band = np.exp(-((f - p) ** 2) / 0.005) + 0.05 * g.random((F, P))
        out[f"monotone{i}"] = (band / band.sum(1, keepdims=True)).astype(np.float32)
    out["short_tokens"] = g.random((6, 20), dtype=np.float32)
    for F in (1, 2, 3, 4):
        out[f"frames{F}"] = g.random((F, 5), dtype=np.float32)
    return out


def main():
    z = {}
    for name, x in cases().items():
        filt = _median_filter(torch.from_numpy(x.T.copy())[None], WIDTH)[0]   # [P, F], along frames
        text, time = _dynamic_time_warping(-filt.double().numpy())
        jumps = np.pad(np.diff(text), (1, 0), constant_values=1).astype(bool)
        z[f"{name}_x"] = x
        z[f"{name}_filtered"] = filt.numpy().T.copy()
        z[f"{name}_jumps"] = time[jumps].astype(np.int32)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "alignment.npz"), **z)


if __name__ == "__main__":
    main()
