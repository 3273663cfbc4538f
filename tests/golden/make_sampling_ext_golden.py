"""Generate tests/golden/sampling_ext.npz by EXECUTING transformers' processors and the reference's ParlerTTSLogitsProcessor.

What is executed (transformers 5.5.0 installed, the stand-in for the pinned 4.46.1 as for warpers.npz):
  * NoRepeatNGramLogitsProcessor, MinPLogitsWarper, TypicalLogitsWarper, EpsilonLogitsWarper, EtaLogitsWarper on fp32 scores
    [6, 1088] (some -inf, some near-ties) and histories [6, 40] with planted repeats
  * GenerationMixin._get_logits_processor on a stub: the processor classes and their order for several knob combinations, with
    the reference's ParlerTTSLogitsProcessor as the merged custom list, and the chain's output
  * the same call for single knob values: which raise ValueError, which add a processor, which are silently off
  * GenerationMixin._prepare_generated_length: the min_length / min_new_tokens / n0 fold
Import shims: those of make_golden.py (the reference's package imports).

Usage:  PARLER_TTS_REFERENCE=<checkout> python tests/golden/make_sampling_ext_golden.py
"""
from __future__ import annotations
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import import_reference  # noqa: E402

R, V, T, K, EOS = 6, 1088, 40, 3, 1024
CHAINS = [
    dict(do_sample=False, no_repeat_ngram_size=2, min_length=45),
    dict(do_sample=True, top_k=50, no_repeat_ngram_size=3, min_p=0.1),
    dict(do_sample=True, temperature=0.7, top_p=0.9, typical_p=0.8),
    dict(do_sample=True, top_k=200, epsilon_cutoff=0.002, eta_cutoff=0.001),
    dict(do_sample=True, temperature=1.3, top_k=100, top_p=0.95, min_p=0.02, typical_p=0.95, epsilon_cutoff=3e-4, eta_cutoff=3e-4,
         no_repeat_ngram_size=1, min_new_tokens=50),
    dict(do_sample=False, min_p=0.5, typical_p=0.5, epsilon_cutoff=0.1, eta_cutoff=0.1),
]
VALIDATION = [("min_p", 1.5), ("min_p", -0.1), ("min_p", 0.0), ("min_p", 1.0), ("typical_p", 0.0), ("typical_p", -1.0),
              ("typical_p", 1.0), ("typical_p", 1.5), ("typical_p", 0.5), ("epsilon_cutoff", 1.5), ("epsilon_cutoff", 0.0),
              ("epsilon_cutoff", 1.0), ("epsilon_cutoff", 0.5), ("eta_cutoff", 1.5), ("eta_cutoff", -0.2), ("eta_cutoff", 0.5),
              ("no_repeat_ngram_size", 2.5), ("no_repeat_ngram_size", -1), ("no_repeat_ngram_size", 0), ("no_repeat_ngram_size", 3),
              ("min_length", 2.5), ("min_length", -3), ("min_length", 0), ("min_length", 7)]
FOLD = [(None, None, 1), (10, None, 1), (10, None, 4), (3, None, 5), (10, 4, 1), (10, 0, 3), (None, 6, 3), (0, None, 2)]


def inputs():
    g = torch.Generator().manual_seed(17)
    scores = torch.randn(R, V, generator=g) * 2.5
    scores[0, 5:40] = -float("inf")
    scores[1, ::7] = -float("inf")
    scores[2, 100:110] = scores[2, 100]                        # a run of ties
    scores[3, 7] = scores[3].max() + 4.0                       # one dominant id
    scores[4] = scores[4] * 0.05                               # nearly flat
    scores[5, 11] = scores[5, 12] = scores[5].max() + 0.5      # tied maxima
    ids = torch.randint(0, 60, (R, T), generator=g)
    ids[:, 0] = 1025
    ids[0, 10:13] = ids[0, 37:40]                              # the last trigram seen before
    ids[1, 3:5] = ids[1, 38:40]
    ids[1, 20:22] = ids[1, 38:40]
    ids[2, 30:33] = ids[2, 38:40].repeat(2)[:3]
    ids[3, :] = 9                                              # one id throughout
    ids[4, 17:20] = ids[4, 37:40]
    return scores, ids


def main():
    import_reference()
    from parler_tts.logits_processors import ParlerTTSLogitsProcessor
    from transformers import GenerationConfig
    from transformers.generation import utils as gu
    from transformers.generation.logits_process import (EpsilonLogitsWarper, EtaLogitsWarper, LogitsProcessorList,
                                                        MinPLogitsWarper, NoRepeatNGramLogitsProcessor, TypicalLogitsWarper)
    scores, ids = inputs()
    out = dict(scores=scores.numpy(), ids=ids.numpy())
    single = {"ngram": (NoRepeatNGramLogitsProcessor, [1, 2, 3, 4, 41]), "min_p": (MinPLogitsWarper, [0.05, 0.3, 1.0]),
              "typical": (TypicalLogitsWarper, [0.2, 0.9, 0.999]), "epsilon": (EpsilonLogitsWarper, [3e-4, 0.01]),
              "eta": (EtaLogitsWarper, [3e-4, 0.02])}
    for name, (cls, vals) in single.items():
        out[f"{name}_values"] = np.array(vals, dtype=np.float64)
        for i, v in enumerate(vals):
            out[f"{name}_{i}"] = cls(v)(ids, scores.clone()).numpy()

    class Stub:  # the attributes of the model the two GenerationMixin methods read
        config = types.SimpleNamespace(is_encoder_decoder=True, max_position_embeddings=None, get_text_config=lambda: None)
        _merge_criteria_processor_list = gu.GenerationMixin._merge_criteria_processor_list
    stub = Stub()

    def processors(knobs, n0=1, parler=None):
        gc = GenerationConfig(eos_token_id=EOS, pad_token_id=1024, bos_token_id=1025, **knobs)
        gc._eos_token_tensor = torch.tensor([EOS])
        custom = LogitsProcessorList([parler] if parler is not None else [])
        return gc, gu.GenerationMixin._get_logits_processor(stub, generation_config=gc, input_ids_seq_length=n0, encoder_input_ids=None,
                                                            logits_processor=custom, device="cpu", model_kwargs={})

    for ci, knobs in enumerate(CHAINS):
        parler = ParlerTTSLogitsProcessor(eos_token_id=EOS, num_codebooks=K, batch_size=R // K, device="cpu")
        gc, procs = processors(knobs, parler=parler)
        out[f"chain{ci}_knobs"] = np.array(json.dumps(knobs))
        out[f"chain{ci}_order"] = np.array(json.dumps([type(p).__name__ for p in procs]))
        s = scores.clone()
        for p in procs:
            s = p(ids, s)
        out[f"chain{ci}_out"] = s.numpy()
    # 0: no processor, 1: a processor, 2: ValueError (do_sample=True so that the warpers are built)
    status = []
    for knob, v in VALIDATION:
        try:
            _, procs = processors({knob: v, "do_sample": True, "top_k": None})
            status.append(1 if len(procs) else 0)
        except ValueError:
            status.append(2)
    out["validation"] = np.array(json.dumps([[k, v, s] for (k, v), s in zip(VALIDATION, status)]))
    fold = []
    for ml, mnt, n0 in FOLD:
        kw = {} if ml is None else dict(min_length=ml)
        if mnt is not None:
            kw["min_new_tokens"] = mnt
        gc = GenerationConfig(eos_token_id=EOS, max_length=100, **kw)
        gu.GenerationMixin._prepare_generated_length(stub, gc, has_default_max_length=False, has_default_min_length=ml is None,
                                                     model_input_name="input_ids", input_ids_length=n0, inputs_tensor=None)
        fold.append([ml, mnt, n0, gc.min_length])
    out["fold"] = np.array(json.dumps(fold))
    np.savez_compressed(os.path.join(HERE, "sampling_ext.npz"), **out)
    print("wrote sampling_ext.npz:", sorted(out))


if __name__ == "__main__":
    main()
