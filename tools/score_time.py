"""Time teacher-forced scoring (ParlerTTSForConditionalGeneration.forward(labels=...)) at the Mini shape, bf16.

B = 32 utterances, S = 64 description positions, P = 32 prompt positions, T = 86 / 430 / 1720 frames (1 / 5 / 20 s of audio),
24 layers with synthetic weights.  Per T it prints:
  * forward(labels=...) on the fused heads + cross-entropy kernel: host clock around a device synchronise, median of 5;
  * the same with return_logits=True (the unfused route, which writes the [B*K, T, V] fp32 logits);
  * ce_fused_kernel alone: its device time from a torch.profiler trace of 5 calls (mean per call), and its rate over the
    heads' 2*B*T*H*K*V operations.
The card's name, power limit and max SM clock are read in the same run.

    python tools/score_time.py [--T 86 430 1720] [--reps 5] [--json out.json]
"""
from __future__ import annotations
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover - reported, not fatal
        q = f"unknown ({e!r})"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, nargs="+", default=[86, 430, 1720])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("score_time.py measures on the GPU; no CUDA device is visible")
    from oracle.config import mini_cfg, tiny_dac_cfg
    from oracle.weights import make_dac_weights, make_decoder_weights
    from tests.helpers import build_product_model, synth_inputs
    cfg = mini_cfg()
    w = make_decoder_weights(cfg, seed=1, head_std=0.1)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=torch.bfloat16)
    B, S, P, K, V, H = 32, 64, 32, cfg.num_codebooks, cfg.vocab_size, cfg.hidden_size
    rows = []
    gpu = card()
    print(f"card: {gpu}")
    for T in a.T:
        enc, em, prompt, pm = synth_inputs(cfg, B, S, P, seed=T)
        g = torch.Generator().manual_seed(T)
        labels = torch.randint(0, 1024, (B, T, K), generator=g)
        args = dict(encoder_outputs=(enc.cuda(),), attention_mask=em.cuda(), prompt_hidden_states=prompt.cuda(),
                    prompt_attention_mask=pm.cuda(), labels=labels.cuda())

        def timed(**kw):
            model(**args, **kw)
            torch.cuda.synchronize()
            ts = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                model(**args, **kw)
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
            return sorted(ts)[len(ts) // 2] * 1e3

        fused_ms = timed()
        logits_ms = timed(return_logits=True)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                model(**args)
            torch.cuda.synchronize()
        k_us = sum(e.device_time_total for e in prof.key_averages() if "ce_fused_kernel" in e.key) / a.reps
        g_us = sum(e.device_time_total for e in prof.key_averages() if "gather_label_rows_kernel" in e.key) / a.reps
        flop = 2.0 * B * T * H * K * V
        r = dict(T=T, forward_ms=fused_ms, forward_return_logits_ms=logits_ms, ce_fused_kernel_ms=k_us / 1e3,
                 gather_rows_ms=g_us / 1e3, heads_tflop=flop / 1e12, ce_fused_tflops=flop / (k_us * 1e-6) / 1e12 if k_us else None)
        rows.append(r)
        print(f"T={T:5d}: forward(labels) {fused_ms:8.2f} ms | return_logits=True {logits_ms:8.2f} ms | ce_fused_kernel "
              f"{k_us / 1e3:7.3f} ms ({r['ce_fused_tflops'] or 0:6.1f} TFLOP/s over {flop / 1e12:.3f} TFLOP) | row gather {g_us / 1e3:.3f} ms")
    out = dict(card=gpu, B=B, S=S, P=P, rows=rows)
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
