"""Time generate()'s token loop with output_attentions + output_hidden_states against the default path, at Mini, B = 1 and 32.

Mini (24 layers, synthetic weights), bf16, S = 64, P = 32, 128 decode steps (max_length 129, min_new_tokens 128 so every run has
the same length), top_k = 50 sampling.  Per batch size the calls run alternated, three rounds; each time is a host clock around a
device synchronise (decoder token loop only), and the median, the spread (max - min over the median) and the per-step time are
printed.
  * default                                    the cluster kernel, up to 64 tokens per launch (the decoder's default path)
  * multi-kernel path (PTTS_FUSED=0)           the path a probe window switches to, without the probe kernels
  * output_attentions + output_hidden_states   the multi-kernel graph with the probe kernels, writing into 64-step chunks
The card's name, power limit and max SM clock are read in the same run.

    python tools/probe_time.py [--reps 3] [--json out.json]
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
from tools.score_time import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("probe_time.py measures on the GPU; no CUDA device is visible")
    from oracle.config import mini_cfg, tiny_dac_cfg
    from oracle.weights import make_dac_weights, make_decoder_weights
    from parler_tts_b200.configuration import GenerationConfig
    from parler_tts_b200.modeling import StepProbes
    from tests.helpers import build_product_model, synth_inputs
    cfg = mini_cfg()
    w = make_decoder_weights(cfg, seed=1, head_std=0.1)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=torch.bfloat16)
    S, P, steps = 64, 32, 128
    L = steps + 1
    gpu = card()
    print(f"card: {gpu}")
    rows = []
    for B in (1, 32):
        enc, em, prompt, pm = synth_inputs(cfg, B, S, P, seed=0)
        enc, prompt = enc.cuda().bfloat16(), prompt.cuda().bfloat16()
        em, pm = em.cuda(), pm.cuda()
        sampling = model._sampling(GenerationConfig(do_sample=True, top_k=50, max_length=L, min_new_tokens=steps), 1, L, seed=1)

        def loop(mode):
            probe = mode == "probes"
            if mode == "multi":
                os.environ["PTTS_FUSED"] = "0"   # read when the session picks its path at the prefill
            rec = StepProbes(cfg.num_hidden_layers, B, cfg.num_attention_heads, S, cfg.hidden_size, P, 1, torch.bfloat16,
                             model.device, True, True) if probe else None
            try:
                ids = model._run_token_loop(enc, em, prompt, pm, None, sampling, (0, B, 0, B), [rec] if probe else [])
            finally:
                os.environ.pop("PTTS_FUSED", None)
            return ids, rec

        modes = {"default": "default", "multi": "multi-kernel path (PTTS_FUSED=0)",
                 "probes": "output_attentions + output_hidden_states"}
        for mode in modes:   # warm-up: modules, graphs, the session
            loop(mode)
        times = {m: [] for m in modes}
        ref = None
        for _ in range(a.reps):
            for mode in modes:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ids, rec = loop(mode)
                torch.cuda.synchronize()
                times[mode].append(time.perf_counter() - t0)
                ref = ids if ref is None else ref
                assert torch.equal(ids, ref), f"{modes[mode]}: the token ids differ from the default path's"
                del rec
        for mode, ts in times.items():
            med = statistics.median(ts)
            name = modes[mode]
            rows.append(dict(B=B, call=name, ms=1e3 * med, us_per_step=1e6 * med / steps, spread=(max(ts) - min(ts)) / med))
            print(f"B={B:2d} {name:42s} {1e3 * med:9.2f} ms  {1e6 * med / steps:8.1f} us/step  spread {rows[-1]['spread']:.3f}")
        mb = 2 * cfg.num_hidden_layers * B * cfg.num_attention_heads * sum(P + 1 + t for t in range(1, steps + 1)) / 1e6
        print(f"B={B:2d} self-attention weights recorded over the {steps} steps: {mb:.1f} MB")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=gpu, rows=rows, shape=dict(S=S, P=P, steps=steps)), f, indent=1)


if __name__ == "__main__":
    main()
