"""Codes -> waveform time of a batch of utterances of different lengths: generate()'s former per-sample loop against one ragged
DACModel.decode(frame_lengths=...) call, with the padded equal-length batch for scale.

44.1 kHz DAC (DACConfig(), synthetic weights), bf16, B = 32, each row n_b frames drawn from a seed uniformly in [T/4, T] and
then EOS (1024) up to T, as generate() leaves a batch whose utterances end at different frames; T = 248 and 1016 (the 256- and
1024-step configs).  Timed, alternated, --reps rounds after one warm-up round:
  * loop:    the parent's per-sample branch of generate() -- per row a host-synchronising valid count, a boolean frame gather,
             a batch-1 decode, then pad_sequence; host clock around a device synchronise;
  * ragged:  one decode(frame_lengths=n) over the frames already packed to the front; CUDA events and the host clock;
  * padded:  decode of a full-length [32, K, T] batch (every frame valid); CUDA events;
  * step:    modeling.codes_to_waveform on the same EOS-padded codes (compaction + one ragged call + lengths), host clock.
The outputs of loop, ragged and step are checked equal.  Median and spread (max - min over the median) are printed with the card's
name, power limit and max SM clock read in the same run.

    python tools/dac_ragged_time.py [--T 248 1016] [--reps 5] [--json out.json]
"""
from __future__ import annotations
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from tools.score_time import card  # noqa: E402


def per_sample_loop(dac, codes, cs, dtype):
    """generate()'s codes -> waveform branch before the ragged decode: one batch-1 decode per row."""
    outs = []
    for b in range(codes.shape[0]):
        sample = codes[None, b]
        ok = (sample >= cs).sum(dim=(0, 1)) == 0
        if int(ok.sum()) > 0:
            outs.append(dac.decode(audio_codes=sample[:, :, ok][None], audio_scales=[None]).audio_values.reshape(-1))
        else:
            outs.append(torch.zeros(1, device=codes.device, dtype=dtype))
    return torch.nn.utils.rnn.pad_sequence(outs, batch_first=True, padding_value=0), [o.shape[0] for o in outs]


def stats(xs):
    med = statistics.median(xs)
    return {"median_ms": round(med, 3), "spread": round((max(xs) - min(xs)) / med, 4), "runs_ms": [round(x, 3) for x in xs]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, nargs="+", default=[248, 1016])
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dac_ragged_time.py measures on the GPU; no CUDA device is visible")
    from parler_tts_b200 import DACConfig, DACModel
    from parler_tts_b200.modeling import codes_to_waveform
    dev = torch.device("cuda", 0)
    cfg = DACConfig()
    dac = DACModel(cfg, dev, torch.bfloat16).load_state_dict(bench.synth_dac_weights(cfg, dev))
    cs, K, B = cfg.codebook_size, cfg.num_codebooks, a.B
    result = {"card": card(), "B": B, "dtype": "bf16", "codec": "DACConfig() 44.1 kHz", "configs": []}
    for T in a.T:
        g = torch.Generator().manual_seed(1000 + T)
        n = torch.randint(T // 4, T + 1, (B,), generator=g)
        full = torch.randint(0, cs, (B, K, T), generator=g).to(dev)
        eos = full.clone()
        for b in range(B):
            eos[b, :, int(n[b]):] = cs
        n_list = n.tolist()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def host(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3, out

        def events(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ev0.record()
            out = fn()
            ev1.record()
            torch.cuda.synchronize()
            return ev0.elapsed_time(ev1), (time.perf_counter() - t0) * 1e3, out

        runs = {k: [] for k in ("loop", "ragged_events", "ragged_host", "padded_events", "step")}
        outs = {}
        for rep in range(a.reps + 1):   # round 0 warms every shape up
            t, outs["loop"] = host(lambda: per_sample_loop(dac, eos, cs, torch.bfloat16))
            te, th, outs["ragged"] = events(lambda: dac.decode(eos[None], [None] * B, frame_lengths=n_list).audio_values)
            tp, _, _ = events(lambda: dac.decode(full[None], [None] * B).audio_values)
            ts, outs["step"] = host(lambda: codes_to_waveform(dac, eos, cs, torch.bfloat16))
            if rep > 0:
                runs["loop"].append(t); runs["ragged_events"].append(te); runs["ragged_host"].append(th)
                runs["padded_events"].append(tp); runs["step"].append(ts)
        loop_audio, loop_len = outs["loop"]
        step_audio, step_len = outs["step"]
        width = loop_audio.shape[1]
        same = (torch.equal(loop_audio, step_audio) and loop_len == step_len
                and torch.equal(outs["ragged"].squeeze(1)[:, :width], loop_audio))
        row = {"T": T, "frames": sum(n_list), "frames_padded": B * T, "outputs_equal": bool(same)}
        row.update({k: stats(v) for k, v in runs.items()})
        row["loop_over_ragged_host"] = round(row["loop"]["median_ms"] / row["ragged_host"]["median_ms"], 2)
        row["loop_over_step"] = round(row["loop"]["median_ms"] / row["step"]["median_ms"], 2)
        result["configs"].append(row)
        print(json.dumps(row), flush=True)
        if not same:
            raise SystemExit(f"T={T}: the ragged decode and the per-sample loop differ")
    print(json.dumps({"card": result["card"]}))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
