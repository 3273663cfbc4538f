"""Time generate()'s token loop with output_scores + output_logits against the default path and the split path, at bench config
1's shapes.

Mini (24 layers, synthetic weights), bf16, B = 32, S = 64, P = 32, 256 decode steps (max_length 257, min_new_tokens 256 so every
run has the same length), top_k = 50 sampling.  The calls below run alternated, five rounds; each time is a host clock around a
device synchronise (decoder token loop only: the codes, not the waveform), and the median and the spread (max - min over the
median) are printed.
  * default                               the cluster kernel, up to 64 tokens per launch
  * no_repeat_ngram_size = max_length + 1 the split path alone: step kernel without its sampling phase + EXT sampler per token
  * output_scores + output_logits         the split path, the sampler also writing both rows of every step into 64-step chunks
The card's name, power limit and max SM clock are read in the same run.

    python tools/generate_outputs_time.py [--reps 5] [--json out.json]
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
        raise SystemExit("generate_outputs_time.py measures on the GPU; no CUDA device is visible")
    from oracle.config import mini_cfg, tiny_dac_cfg
    from oracle.weights import make_dac_weights, make_decoder_weights
    from parler_tts_b200.configuration import GenerationConfig
    from parler_tts_b200.modeling import StepOutputs
    from tests.helpers import build_product_model, synth_inputs
    cfg = mini_cfg()
    w = make_decoder_weights(cfg, seed=1, head_std=0.1)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=torch.bfloat16)
    B, S, P, steps = 32, 64, 32, 256
    L = steps + 1
    K, V = cfg.num_codebooks, cfg.vocab_size
    enc, em, prompt, pm = synth_inputs(cfg, B, S, P, seed=0)
    base = dict(encoder_outputs=(enc.cuda().bfloat16(),), attention_mask=em.cuda(), prompt_hidden_states=prompt.cuda().bfloat16(),
                prompt_attention_mask=pm.cuda(), do_sample=True, top_k=50, max_length=L, min_new_tokens=steps, seed=1)
    calls = {"default": ({}, False), "split path (ngram = max_length + 1)": (dict(no_repeat_ngram_size=L + 1), False),
             "output_scores + output_logits": ({}, True)}

    def codes_only(extra, outputs):
        # generate()'s token loop without the DAC decode; with outputs, the storage generate() would pass
        gc = GenerationConfig(**{k: v for k, v in {**base, **extra}.items() if k in GenerationConfig().__dict__})
        rec = StepOutputs(B * K, V, model.device, True, True) if outputs else None
        ids = model._run_token_loop(base["encoder_outputs"][0], base["attention_mask"], base["prompt_hidden_states"],
                                    base["prompt_attention_mask"], None, model._sampling(gc, 1, L, seed=1), (0, B, 0, B),
                                    [rec] if outputs else [])
        return ids, rec

    gpu = card()
    print(f"card: {gpu}")
    for extra, outputs in calls.values():   # warm-up: modules, graphs, the session
        codes_only(extra, outputs)
    torch.cuda.synchronize()
    times = {k: [] for k in calls}
    ref = None
    for _ in range(a.reps):
        for name, (extra, outputs) in calls.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ids, rec = codes_only(extra, outputs)
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
            assert ids.shape[1] == L, (name, ids.shape)
            ref = ids if ref is None else ref
            assert torch.equal(ids, ref), f"{name}: the token ids differ from the default path's"
            if rec is not None:
                r = rec.result(steps)
                assert len(r["scores"]) == steps and not torch.isnan(r["scores"][-1]).any()
            del rec
    rows = []
    t_def = statistics.median(times["default"])
    t_split = statistics.median(times["split path (ngram = max_length + 1)"])
    for name, ts in times.items():
        med = statistics.median(ts)
        rows.append(dict(call=name, ms=1e3 * med, us_per_step=1e6 * med / steps, vs_default=med / t_def, vs_split=med / t_split,
                         spread=(max(ts) - min(ts)) / med))
        print(f"{name:40s} {1e3 * med:9.2f} ms  {1e6 * med / steps:8.1f} us/step  x{med / t_def:.3f} of default  "
              f"x{med / t_split:.3f} of split  spread {rows[-1]['spread']:.3f}")
    mb = 2 * B * K * V * 4 / 1e6
    print(f"output rows written per step: {mb:.2f} MB ({mb / 2:.2f} MB each)")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=gpu, rows=rows, shape=dict(B=B, S=S, P=P, steps=steps), mb_per_step=mb), f, indent=1)


if __name__ == "__main__":
    main()
