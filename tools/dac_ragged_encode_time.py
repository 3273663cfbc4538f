"""Waveform -> codes time of a batch of clips of different lengths: generate()'s former per-length loop of DACModel.encode calls
against one ragged DACModel.encode(sample_lengths=...) call.

44.1 kHz DAC (DACConfig() shape, synthetic encoder weights), bf16, wgmma path, B = 32 clips whose lengths are drawn from a seed
uniformly in [1 s, 20 s] (samples).  Timed with CUDA events, alternated, --reps rounds after one warm-up round:
  * loop:    the parent's _encode_clips: one encode per distinct length (here every clip), batch 1 each;
  * ragged:  one encode over the clips right-padded to the longest, sample_lengths = their lengths;
  * padded:  encode of the same padded batch without lengths (every row encoded to the longest), for scale.
Each clip's codes from the loop and from the ragged call are checked equal.  Median and spread (max - min over the median) are
printed with the card's name, power limit and max SM clock read in the same run.

    python tools/dac_ragged_encode_time.py [--B 32] [--reps 5] [--seed 0] [--json out.json]
"""
from __future__ import annotations
import argparse
import json
import math
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.score_time import card  # noqa: E402


def stats(xs):
    med = statistics.median(xs)
    return {"median_ms": round(med, 3), "spread": round((max(xs) - min(xs)) / med, 4), "runs_ms": [round(x, 3) for x in xs]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dac_ragged_encode_time.py measures on the GPU; no CUDA device is visible")
    from oracle.config import dac_cfg
    from oracle.weights import make_dac_weights
    from tests.dac_encode_oracle import make_dac_encoder_weights
    from parler_tts_b200 import DACConfig, DACModel
    os.environ["PTTS_DAC_TC"] = "1"
    dev = torch.device("cuda", 0)
    cfg = DACConfig()
    w = make_dac_weights(dac_cfg(), seed=3)
    w.update(make_dac_encoder_weights(dac_cfg(), seed=7))
    dac = DACModel(cfg, dev, torch.bfloat16).load_state_dict(w)
    sr, hop, B = cfg.sampling_rate, dac.hop_length, a.B
    g = torch.Generator().manual_seed(a.seed)
    lens = torch.randint(sr, 20 * sr + 1, (B,), generator=g).tolist()
    n = max(lens)
    t = torch.arange(n) / sr
    wav = (0.3 * torch.sin(2 * math.pi * 200.0 * t) + 0.1 * torch.randn(B, n, generator=g)).to(torch.bfloat16)
    for b, nb in enumerate(lens):
        wav[b, nb:] = 0
    wav = wav[:, None, :].to(dev)
    clips = [wav[b:b + 1, :, :nb] for b, nb in enumerate(lens)]

    def loop():
        codes = [None] * B
        for nb in sorted(set(lens)):
            idx = [i for i, m in enumerate(lens) if m == nb]
            c = dac.encode(torch.cat([clips[i] for i in idx])).audio_codes[0]
            for j, i in enumerate(idx):
                codes[i] = c[j]
        return codes

    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def events(fn):
        torch.cuda.synchronize()
        ev0.record()
        out = fn()
        ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1), out

    runs = {k: [] for k in ("loop", "ragged", "padded")}
    outs = {}
    for rep in range(a.reps + 1):   # round 0 warms every shape up
        tl, outs["loop"] = events(loop)
        tr, outs["ragged"] = events(lambda: dac.encode(wav, sample_lengths=lens).audio_codes[0])
        tp, _ = events(lambda: dac.encode(wav).audio_codes[0])
        if rep > 0:
            runs["loop"].append(tl); runs["ragged"].append(tr); runs["padded"].append(tp)
    rag = outs["ragged"]
    same = all(torch.equal(rag[b, :, :math.ceil(nb / hop)], outs["loop"][b]) for b, nb in enumerate(lens))
    same = same and all(bool((rag[b, :, math.ceil(nb / hop):] == cfg.codebook_size).all()) for b, nb in enumerate(lens))
    result = {"card": card(), "B": B, "dtype": "bf16", "codec": "DACConfig() 44.1 kHz, wgmma path", "seed": a.seed,
              "clip_seconds": {"min": round(min(lens) / sr, 3), "median": round(statistics.median(lens) / sr, 3),
                               "max": round(n / sr, 3), "total": round(sum(lens) / sr, 3)},
              "distinct_lengths": len(set(lens)), "frames": sum(math.ceil(nb / hop) for nb in lens),
              "frames_padded": B * math.ceil(n / hop), "outputs_equal": bool(same)}
    result.update({k: stats(v) for k, v in runs.items()})
    result["loop_over_ragged"] = round(result["loop"]["median_ms"] / result["ragged"]["median_ms"], 2)
    result["card_after"] = card()
    print(json.dumps(result), flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)
    if not same:
        raise SystemExit("the ragged encode and the per-length loop differ")


if __name__ == "__main__":
    main()
