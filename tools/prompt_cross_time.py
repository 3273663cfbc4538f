"""Decode-step time with the transcript prompt as cross-attention keys (config.prompt_cross_attention) against the prompt as a
self-attention prefix, at the same prompt length P.

Mini (24 layers, synthetic weights), bf16, B = 32, S = 64 description keys, P = 32 / 128 / 448.  One decoder engine serves both
layouts, since the step kernels do not know the config flag:
  * prefix  session (B, P, S):      P + n self-attention keys at step n, S cross keys
  * cross   session (B, 0, S + P):  n self-attention keys, S + P cross keys (prompt_cross_states, as generate() builds them)
Per layout: prefill, the first sample, then 128 decode steps in one ptts_decode_steps call between CUDA events (top_k = 50
sampling, min_new_tokens so every run has the same length).  The layouts run alternated, --reps rounds after one warm-up round
each; the median and the spread (max - min over the median) of the per-step time are printed with the decode path, and the
card's name, power limit and max SM clock are read in the same run.

    python tools/prompt_cross_time.py [--P 32 128 448] [--reps 5] [--json out.json]
"""
from __future__ import annotations
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from tools.score_time import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, nargs="+", default=[32, 128, 448])
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prompt_cross_time.py measures on the GPU; no CUDA device is visible")
    from parler_tts_b200 import DACConfig, ParlerTTSConfig, ParlerTTSDecoderConfig, ParlerTTSForConditionalGeneration
    from parler_tts_b200.modeling import GenSession, _sinusoidal_table, prompt_cross_states
    dev = torch.device("cuda", 0)
    cfg = ParlerTTSConfig(vocab_size=32128, text_encoder={}, audio_encoder=DACConfig(), decoder=ParlerTTSDecoderConfig(**bench.MINI))
    model = ParlerTTSForConditionalGeneration(cfg, device=dev, dtype=torch.bfloat16)
    model.load_state_dict(bench.synthetic_state_dict(bench.MINI, dev))
    eng = model.decoder.engine
    B, S, n = 32, bench.S_LEN, a.steps
    L = n + 1
    gen = dict(do_sample=True, top_k=50, min_new_tokens=n, suppress_special=True, codebook_size=1024)
    positions = _sinusoidal_table(bench.MINI["max_position_embeddings"], bench.MINI["hidden_size"]).to(dev, torch.bfloat16)
    results = {"card": card(), "B": B, "S": S, "decode_steps": n - 1, "rows": []}
    print(f"[prompt-cross] {results['card']}; Mini bf16, B = {B}, S = {S}, {n - 1} timed decode steps per run", flush=True)
    for P in a.P:
        g = torch.Generator().manual_seed(P)
        enc, em, _, _ = bench.synthetic_inputs(B, bench.MINI["hidden_size"], seed=P, device=dev)
        ids = torch.randint(0, 32128, (B, P), generator=g).to(dev)
        pm = torch.ones(B, P, dtype=torch.long)
        for b, ln in enumerate(torch.randint(P // 2, P + 1, (B,), generator=g).tolist()):
            pm[b, : P - ln] = 0
        pm = pm.to(dev)
        prompt = torch.nn.functional.embedding(ids, model.embed_prompts_weight)   # the prefix layout's prompt states
        states, mask = prompt_cross_states(enc, em, ids, pm, model.embed_prompts_weight, positions)
        layouts = {"prefix": (GenSession(eng, B, P, S, P + L), (prompt, pm, enc, em)),
                   "cross": (GenSession(eng, B, 0, S + P, L), (None, None, states, mask))}

        def run(name):
            sess, args = layouts[name]
            sess.begin(L, seed=1, **gen)
            sess.prefill(*args)
            sess.sample()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            sess.decode_steps(n - 1)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / (n - 1) * 1e3   # us per step

        for name in layouts:
            run(name)   # warm-up: graph capture and first launches
        times = {name: [] for name in layouts}
        for _ in range(a.reps):
            for name in layouts:
                times[name].append(run(name))
        row = {"P": P}
        for name, ts in times.items():
            med = statistics.median(ts)
            row[name] = dict(us_per_step=med, spread=(max(ts) - min(ts)) / med, path=layouts[name][0].fused)
        row["cross_over_prefix"] = row["cross"]["us_per_step"] / row["prefix"]["us_per_step"]
        results["rows"].append(row)
        print(f"[prompt-cross] P = {P:4d}: prefix {row['prefix']['us_per_step']:7.1f} us/step (spread {row['prefix']['spread']:.1%}, "
              f"path {row['prefix']['path']}), cross {row['cross']['us_per_step']:7.1f} us/step (spread {row['cross']['spread']:.1%}, "
              f"path {row['cross']['path']}): cross / prefix = {row['cross_over_prefix']:.3f}", flush=True)
        for sess, _ in layouts.values():
            sess.close()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
