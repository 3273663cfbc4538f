"""Time generate()'s token loop with return_token_timestamps against the default path, and the median filter + DTW, at Mini
bf16, B = 32, P = 32, for 256 and 1024 decode steps.

Mini (24 layers, synthetic weights), S = 64, P = 32 transcript tokens, top_k = 50 sampling, min_new_tokens = steps so every run
has the same length.  Per length the calls run alternated, three rounds; each time is a host clock around a device synchronise
(decoder token loop only), and the median, the spread (max - min over the median) and the per-step time are printed.
  * default                          the cluster kernel, up to 64 tokens per launch (the decoder's default path)
  * multi-kernel path (PTTS_FUSED=0) the path an alignment window switches to, without the alignment kernels
  * return_token_timestamps          the multi-kernel graph with the alignment kernels of the default heads (the 192 heads of
                                     layers 12 .. 23), writing one [32, 32] row per step
  * align_dtw                        ptts_align_dtw over the [32, steps, 32] alignment (CUDA events, 20 calls)
The card's name, power limit and max SM clock are read in the same run.

    python tools/timestamps_time.py [--reps 3] [--json out.json]
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
        raise SystemExit("timestamps_time.py measures on the GPU; no CUDA device is visible")
    from oracle.config import mini_cfg, tiny_dac_cfg
    from oracle.weights import make_dac_weights, make_decoder_weights
    from parler_tts_b200.configuration import GenerationConfig
    from parler_tts_b200.modeling import StepAlignment, align_dtw, resolve_alignment_heads
    from tests.helpers import build_product_model, synth_inputs
    cfg = mini_cfg()
    w = make_decoder_weights(cfg, seed=1, head_std=0.1)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=torch.bfloat16)
    B, S, P = 32, 64, 32
    heads = resolve_alignment_heads(None, cfg.num_hidden_layers, cfg.num_attention_heads)
    gpu = card()
    print(f"card: {gpu}")
    enc, em, prompt, pm = synth_inputs(cfg, B, S, P, seed=0)
    enc, prompt, em, pm = enc.cuda().bfloat16(), prompt.cuda().bfloat16(), em.cuda(), pm.cuda()
    rows = []
    for steps in (256, 1024):
        L = steps + 1
        sampling = model._sampling(GenerationConfig(do_sample=True, top_k=50, max_length=L, min_new_tokens=steps), 1, L, seed=1)

        def loop(mode):
            if mode == "multi":
                os.environ["PTTS_FUSED"] = "0"   # read when the session picks its path at the prefill
            rec = StepAlignment(heads, B, L - 1, 0, P, model.device) if mode == "align" else None
            try:
                ids = model._run_token_loop(enc, em, prompt, pm, None, sampling, (0, B, 0, B), [] if rec is None else [rec])
            finally:
                os.environ.pop("PTTS_FUSED", None)
            return ids, rec

        modes = {"default": "default", "multi": "multi-kernel path (PTTS_FUSED=0)", "align": "return_token_timestamps"}
        for mode in modes:   # warm-up: modules, graphs, the session
            loop(mode)
        times = {m: [] for m in modes}
        ref, rec_keep = None, None
        for _ in range(a.reps):
            for mode in modes:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ids, rec = loop(mode)
                torch.cuda.synchronize()
                times[mode].append(time.perf_counter() - t0)
                ref = ids if ref is None else ref
                assert torch.equal(ids, ref), f"{modes[mode]}: the token ids differ from the default path's"
                rec_keep = rec if rec is not None else rec_keep
        for mode, ts in times.items():
            med = statistics.median(ts)
            rows.append(dict(steps=steps, call=modes[mode], ms=1e3 * med, us_per_step=1e6 * med / steps, spread=(max(ts) - min(ts)) / med))
            print(f"steps={steps:4d} {modes[mode]:34s} {1e3 * med:9.2f} ms  {1e6 * med / steps:8.1f} us/step  spread {rows[-1]['spread']:.3f}")
        al = rec_keep.alignment[:, :steps - 1].contiguous()
        assert torch.isfinite(al).all()
        nf = torch.full((B,), steps - 1, dtype=torch.int32, device=model.device)
        for _ in range(3):
            align_dtw(al, nf, pm)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            align_dtw(al, nf, pm)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 20
        rows.append(dict(steps=steps, call="align_dtw", ms=ms))
        print(f"steps={steps:4d} {'align_dtw (median filter + DTW)':34s} {ms:9.3f} ms per call, {steps - 1} frames x {P} keys x {B}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=gpu, rows=rows, shape=dict(B=B, S=S, P=P, heads=len(heads))), f, indent=1)


if __name__ == "__main__":
    main()
