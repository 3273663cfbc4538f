"""Time generate() with the ptts_logits_ext processors against the default path: Mini, bf16, B = 32.

Mini (24 layers, synthetic weights), bf16, B = 32, S = 64, P = 32, 256 decode steps (max_length 257, min_new_tokens 256 so
every run has the same length), top_k = 50 sampling.  The calls below run alternated, five rounds; each time is a host clock
around a device synchronise (decoder only: the codes, not the waveform), and the median is printed with its per-token cost.
  * default                                the cluster kernel, up to 64 tokens per launch
  * suppress_tokens                        the split path with a mask stage only (it joins the single mask pass)
  * sequence_bias + decay + renormalize    the ordered per-id pass (an additive stage), and LogitNormalization
  * every stage                            sequence_bias (single and multi-id), suppress, begin-suppress, InfNan, the decay,
                                           forced EOS and renormalize_logits
A separate torch.profiler run of the last call gives the EXT sampler's device time per token and the step kernel's.  The card's
name, power limit and max SM clock are read in the same run.

    python tools/logits_ext_time.py [--reps 5] [--json out.json]
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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("logits_ext_time.py measures on the GPU; no CUDA device is visible")
    from oracle.config import mini_cfg, tiny_dac_cfg
    from oracle.weights import make_dac_weights, make_decoder_weights
    from tests.helpers import build_product_model, synth_inputs
    cfg = mini_cfg()
    w = make_decoder_weights(cfg, seed=1, head_std=0.1)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=torch.bfloat16)
    B, S, P, steps = 32, 64, 32, 256
    L = steps + 1
    enc, em, prompt, pm = synth_inputs(cfg, B, S, P, seed=0)
    base = dict(encoder_outputs=(enc.cuda().bfloat16(),), attention_mask=em.cuda(), prompt_hidden_states=prompt.cuda().bfloat16(),
                prompt_attention_mask=pm.cuda(), do_sample=True, top_k=50, max_length=L, min_new_tokens=steps, seed=1)
    V = cfg.vocab_size
    calls = {"default": {}, "suppress_tokens": dict(suppress_tokens=[V - 1, 7]),
             "sequence_bias + decay + renormalize": dict(sequence_bias={(7,): -1.0, (3, 7): 0.5}, exponential_decay_length_penalty=(200, 1.01),
                                                         renormalize_logits=True),
             "every stage": dict(sequence_bias={(7,): -1.0, (3, 7): 0.5, (5, 9, 7): 0.25}, suppress_tokens=[V - 1],
                                 begin_suppress_tokens=[V - 2], remove_invalid_values=True, exponential_decay_length_penalty=(200, 1.01),
                                 forced_eos_token_id=cfg.eos_token_id, renormalize_logits=True)}
    dec = model.decoder.engine

    def codes_only(extra):
        # generate()'s token loop without the DAC decode: the part the processors change
        from parler_tts_b200.configuration import GenerationConfig
        gc = GenerationConfig(**{k: v for k, v in {**base, **extra}.items() if k in GenerationConfig().__dict__})
        return model._run_token_loop(base["encoder_outputs"][0], base["attention_mask"], base["prompt_hidden_states"],
                                     base["prompt_attention_mask"], None, model._sampling(gc, 1, L, seed=1), (0, B, 0, B))

    gpu = card()
    print(f"card: {gpu}")
    for extra in calls.values():   # warm-up: modules, graphs, the session
        codes_only(extra)
    torch.cuda.synchronize()
    times = {k: [] for k in calls}
    for _ in range(a.reps):
        for name, extra in calls.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = codes_only(extra)
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
            assert out.shape[1] == L, (name, out.shape)
    rows = []
    t_def = statistics.median(times["default"])
    for name, ts in times.items():
        med = statistics.median(ts)
        rows.append(dict(call=name, ms=1e3 * med, us_per_token=1e6 * med / steps, extra_us_per_token=1e6 * (med - t_def) / steps,
                         vs_default=med / t_def, spread=(max(ts) - min(ts)) / med))
        print(f"{name:40s} {1e3 * med:9.2f} ms  {rows[-1]['us_per_token']:8.1f} us/token  {rows[-1]['extra_us_per_token']:+7.1f} "
              f"us/token vs default  x{med / t_def:.3f}  spread {rows[-1]['spread']:.3f}")
    # device time per token of the split path's kernels
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        codes_only(calls["every stage"])
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        if "sample_kernel" in ev.key or "decode_step" in ev.key:
            per[ev.key] = dict(count=ev.count, us_per_call=ev.device_time_total / max(1, ev.count))
            print(f"{ev.key[:90]:90s} {ev.count:5d} calls  {per[ev.key]['us_per_call']:8.2f} us/call")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=gpu, rows=rows, kernels=per, shape=dict(B=B, S=S, P=P, steps=steps)), f, indent=1)


if __name__ == "__main__":
    main()
