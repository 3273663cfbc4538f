"""Decode-step and prefill time of 32 rows as B = 32 / N descriptions x N takes sharing one cross-attention K/V per description
(generate(num_return_sequences=N), ptts_session_create3) against the same 32 rows as the hand-expanded batch (one K/V per row).

Mini (24 layers, synthetic weights), bf16, S = 64 and 256 description keys, N = 1 / 2 / 4 / 8.  Per layout: prefill between CUDA
events, the first sample, then 128 decode steps in one ptts_decode_steps call between CUDA events (top_k = 50 sampling,
min_new_tokens so every run has the same length).  The two layouts run alternated, --reps rounds after one warm-up round each;
the median and the spread (max - min over the median) are printed with the decode path and the cross-K/V workspace bytes
(L + 1 layer strides: the projection's output buffer and the L layers' K/V), and the card's name, power limit and max SM clock
are read in the same run.

    python tools/return_sequences_time.py [--S 64 256] [--N 1 2 4 8] [--reps 5] [--json out.json]
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
    ap.add_argument("--S", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--N", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("return_sequences_time.py measures on the GPU; no CUDA device is visible")
    from parler_tts_b200 import DACConfig, ParlerTTSConfig, ParlerTTSDecoderConfig, ParlerTTSForConditionalGeneration
    from parler_tts_b200.modeling import GenSession
    dev = torch.device("cuda", 0)
    cfg = ParlerTTSConfig(vocab_size=32128, text_encoder={}, audio_encoder=DACConfig(), decoder=ParlerTTSDecoderConfig(**bench.MINI))
    model = ParlerTTSForConditionalGeneration(cfg, device=dev, dtype=torch.bfloat16)
    model.load_state_dict(bench.synthetic_state_dict(bench.MINI, dev))
    eng = model.decoder.engine
    H, nL = bench.MINI["hidden_size"], bench.MINI["num_hidden_layers"]
    ckv_row_bytes = 2 * bench.MINI.get("num_cross_attention_key_value_heads", bench.MINI["num_attention_heads"]) * 64 * 2
    rows, n = 32, a.steps
    L = n + 1
    gen = dict(do_sample=True, top_k=50, min_new_tokens=n, suppress_special=True, codebook_size=1024)
    results = {"card": card(), "rows": rows, "decode_steps": n - 1, "runs": []}
    print(f"[takes] {results['card']}; Mini bf16, {rows} rows, {n - 1} timed decode steps per run", flush=True)
    for S in a.S:
        for N in a.N:
            B = rows // N
            g = torch.Generator().manual_seed(S * 100 + N)
            em = torch.ones(B, S, dtype=torch.long)
            for b, ln in enumerate(torch.randint(S // 2, S + 1, (B,), generator=g).tolist()):
                em[b, : S - ln] = 0
            enc = (torch.randn(B, S, H, generator=g) * em[..., None]).to(dev, torch.bfloat16)
            em = em.to(dev)
            layouts = {"expanded": (GenSession(eng, rows, 0, S, L), (None, None, enc.repeat_interleave(N, 0), em.repeat_interleave(N, 0))),
                       "shared": (GenSession(eng, rows, 0, S, L, takes=N), (None, None, enc, em))}

            def run(name):
                sess, args = layouts[name]
                sess.begin(L, seed=1, **gen)
                e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                e[0].record()
                sess.prefill(*args)
                e[1].record()
                sess.sample()
                e[2].record()
                sess.decode_steps(n - 1)
                e[3].record()
                torch.cuda.synchronize()
                return e[0].elapsed_time(e[1]) * 1e3, e[2].elapsed_time(e[3]) / (n - 1) * 1e3   # us: prefill, per step

            for name in layouts:
                run(name)   # warm-up: first launches
            times = {name: [] for name in layouts}
            for _ in range(a.reps):
                for name in layouts:
                    times[name].append(run(name))
            row = {"S": S, "N": N, "descriptions": B}
            for name, ts in times.items():
                pre, step = [t[0] for t in ts], [t[1] for t in ts]
                ms, mp = statistics.median(step), statistics.median(pre)
                d = B if name == "shared" else rows
                row[name] = dict(us_per_step=ms, step_spread=(max(step) - min(step)) / ms, prefill_us=mp,
                                 prefill_spread=(max(pre) - min(pre)) / mp, path=layouts[name][0].fused,
                                 cross_kv_bytes=(nL + 1) * d * S * ckv_row_bytes)
            row["step_shared_over_expanded"] = row["shared"]["us_per_step"] / row["expanded"]["us_per_step"]
            row["prefill_shared_over_expanded"] = row["shared"]["prefill_us"] / row["expanded"]["prefill_us"]
            results["runs"].append(row)
            ex, sh = row["expanded"], row["shared"]
            print(f"[takes] S = {S:3d}, N = {N}: step expanded {ex['us_per_step']:7.1f} us (spread {ex['step_spread']:.1%}, path "
                  f"{ex['path']}), shared {sh['us_per_step']:7.1f} us (spread {sh['step_spread']:.1%}, path {sh['path']}): "
                  f"{row['step_shared_over_expanded']:.3f}; prefill {ex['prefill_us']:7.0f} / {sh['prefill_us']:7.0f} us; "
                  f"cross K/V {ex['cross_kv_bytes'] / 2**20:6.1f} / {sh['cross_kv_bytes'] / 2**20:6.1f} MiB", flush=True)
            for sess, _ in layouts.values():
                sess.close()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
