"""Generate tests/golden/logits_ext.npz by EXECUTING transformers' processors and the reference's ParlerTTSLogitsProcessor.

What is executed (transformers 5.5.0 installed, the stand-in for the pinned 4.46.1 as for sampling_ext.npz):
  * SequenceBiasLogitsProcessor (dict and list formats, sequences that share their last id), SuppressTokensLogitsProcessor,
    SuppressTokensAtBeginLogitsProcessor, ExponentialDecayLengthPenalty, ForcedBOSTokenLogitsProcessor,
    ForcedEOSTokenLogitsProcessor, InfNanRemoveLogitsProcessor and LogitNormalization on fp32 scores [6, 1088] holding -inf, NaN
    and +inf, an EOS already at -inf and a row with every id at -inf, with histories [6, 40] that end with some biased
    sequences' prefixes and not with others
  * GenerationMixin._get_logits_processor on a stub: the processor classes and their order for several knob combinations (with
    the reference's ParlerTTSLogitsProcessor as the merged custom list), and the chain's output on a history of `cols` columns
  * the same call, then one call of the chain, for knob values transformers rejects (now or at its first call) or accepts
Import shims: those of make_golden.py (the reference's package imports).

Usage:  PARLER_TTS_REFERENCE=<checkout> python tests/golden/make_logits_ext_golden.py
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
# sequence_bias as given to generate(); the histories below end with (3, 7)'s and (5, 9, 7)'s prefixes in some rows
SEQ_BIAS = {(3, 7): -2.0, (7,): 1.5, (5, 9, 7): 0.75, (11,): -3.25, (8, 9, 12): 4.0, (9, 7): 0.3, (EOS,): 0.5}
SEQ_BIAS_LIST = [[[3, 7], -2.0], [[7], 1.5], [[5, 9, 7], 0.75], [[1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16], 2.0]]
SINGLE = {
    "seq_bias": [dict(sequence_bias=SEQ_BIAS), dict(sequence_bias=SEQ_BIAS_LIST)],
    "suppress": [dict(suppress_tokens=[0, 7, EOS, 1087, 5000])],
    "begin_suppress": [dict(begin_suppress_tokens=[7, 3, EOS], begin_index=T), dict(begin_suppress_tokens=[7], begin_index=T - 1)],
    "decay": [dict(exponential_decay_length_penalty=(10, 1.2), n0=1), dict(exponential_decay_length_penalty=(39, 1.5), n0=1),
              dict(exponential_decay_length_penalty=(5, 0.9), n0=3), dict(exponential_decay_length_penalty=(0, 3.7), n0=2)],
    "forced_bos": [dict(forced_bos_token_id=9, cols=1), dict(forced_bos_token_id=9, cols=T)],
    "forced_eos": [dict(forced_eos_token_id=EOS, max_length=T + 1), dict(forced_eos_token_id=EOS, max_length=T + 2)],
    "infnan": [dict()],
    "normalize": [dict()],
}
# (knobs, history columns, n0): the chains through _get_logits_processor, with ParlerTTSLogitsProcessor merged last
CHAINS = [
    (dict(do_sample=False, sequence_bias=SEQ_BIAS, suppress_tokens=[5, 7], begin_suppress_tokens=[11, 12]), T, T),
    (dict(do_sample=False, remove_invalid_values=True, exponential_decay_length_penalty=(20, 1.3), suppress_tokens=[EOS, 2]), T, 1),
    (dict(do_sample=False, forced_eos_token_id=EOS, max_length=T + 1, remove_invalid_values=True, no_repeat_ngram_size=2), T, 1),
    (dict(do_sample=False, forced_bos_token_id=9, begin_suppress_tokens=[3], sequence_bias={(9,): 1.0}), 1, 1),
    (dict(do_sample=False, forced_bos_token_id=9, begin_suppress_tokens=[3, 4], max_length=100), 2, 1),
    (dict(do_sample=True, top_k=50, temperature=0.8, sequence_bias=SEQ_BIAS_LIST, exponential_decay_length_penalty=(4, 1.05),
          min_new_tokens=50, renormalize_logits=True), T, 1),
    (dict(do_sample=True, top_k=0, top_p=0.9, min_p=0.05, remove_invalid_values=True, renormalize_logits=True,
          suppress_tokens=[1, 2, 3], exponential_decay_length_penalty=(30, 2.0)), T, 3),
    (dict(do_sample=False, sequence_bias=SEQ_BIAS, no_repeat_ngram_size=3, min_new_tokens=45, forced_eos_token_id=EOS,
          max_length=T + 1, remove_invalid_values=True, exponential_decay_length_penalty=(1, 1.5), suppress_tokens=[0],
          begin_suppress_tokens=[1], renormalize_logits=True), T, T),
]
VALIDATION = [
    dict(sequence_bias={}), dict(sequence_bias=[]), dict(sequence_bias=5), dict(sequence_bias={7: 1.0}),
    dict(sequence_bias={(7, -1): 1.0}), dict(sequence_bias={(): 1.0}), dict(sequence_bias={(7,): 1}),
    dict(sequence_bias={(7, 1.5): 1.0}), dict(sequence_bias=[[[7], 1]]), dict(sequence_bias=[[[0, 7], 1.0]]),
    dict(sequence_bias=[[(7,), 1.0]]), dict(sequence_bias={(7, V): 1.0}), dict(sequence_bias={(V + 5,): 1.0}),
    dict(sequence_bias={(0, 7): 1.0}), dict(sequence_bias=[[[3, 7], -1.0], [[7], 2.0]]), dict(sequence_bias={(np.int64(7),): 1.0}),
    dict(forced_eos_token_id=-1), dict(forced_eos_token_id=V), dict(forced_eos_token_id=5), dict(forced_bos_token_id=V),
    dict(forced_bos_token_id=0), dict(suppress_tokens=[]), dict(suppress_tokens=[V + 3]), dict(begin_suppress_tokens=[-2, 4]),
    dict(remove_invalid_values=False), dict(renormalize_logits=False), dict(exponential_decay_length_penalty=(3, 1.0)),
]


def inputs():
    g = torch.Generator().manual_seed(23)
    scores = torch.randn(R, V, generator=g) * 3.0
    scores[0, 100:140] = -float("inf")
    scores[1, EOS] = -float("inf")                              # an EOS already masked
    scores[2, 17] = float("nan")
    scores[2, 19] = float("inf")
    scores[2, 21] = -float("inf")
    scores[3, EOS] = -2.5                                       # a negative EOS score (the decay takes its absolute value)
    scores[4, EOS] = -0.0
    scores[4, 33] = -0.0
    scores[5] = -float("inf")                                   # every id masked
    ids = torch.randint(0, 60, (R, T), generator=g)
    ids[:, 0] = 1025
    ids[0, -1] = 3                                              # (3, 7) completes; (9, 7) does not
    ids[1, -2:] = torch.tensor([5, 9])                          # (5, 9, 7) and (9, 7) complete
    ids[2, -2:] = torch.tensor([8, 9])                          # (8, 9, 12) and (9, 7) complete
    ids[3, -1] = 9                                              # (9, 7) only
    ids[4, -2:] = torch.tensor([4, 9])
    ids[5, -1] = 3
    ids[1, 5] = EOS                                             # the Parler processor's state moves for batch item 0
    return scores, ids


def main():
    import_reference()
    from parler_tts.logits_processors import ParlerTTSLogitsProcessor
    from transformers import GenerationConfig
    from transformers.generation import utils as gu
    from transformers.generation import logits_process as lp
    scores, ids = inputs()
    out = dict(scores=scores.numpy(), ids=ids.numpy())

    def run_single(name, kw):
        kw = dict(kw)
        cols = kw.pop("cols", T)
        h = ids[:, :cols]
        if name == "seq_bias":
            p = lp.SequenceBiasLogitsProcessor(kw["sequence_bias"])
        elif name == "suppress":
            p = lp.SuppressTokensLogitsProcessor(kw["suppress_tokens"])
        elif name == "begin_suppress":
            p = lp.SuppressTokensAtBeginLogitsProcessor(kw["begin_suppress_tokens"], kw["begin_index"])
        elif name == "decay":
            p = lp.ExponentialDecayLengthPenalty(kw["exponential_decay_length_penalty"], EOS, kw["n0"])
        elif name == "forced_bos":
            p = lp.ForcedBOSTokenLogitsProcessor(kw["forced_bos_token_id"])
        elif name == "forced_eos":
            p = lp.ForcedEOSTokenLogitsProcessor(kw["max_length"], kw["forced_eos_token_id"])
        elif name == "infnan":
            p = lp.InfNanRemoveLogitsProcessor()
        else:
            p = lp.LogitNormalization()
        return p(h, scores.clone()).numpy()

    # sequence_bias dicts are stored as their list form ([[ids], bias] pairs, same order)
    enc = lambda kw: json.dumps({k: ([[list(a), b] for a, b in v.items()] if k == "sequence_bias" and isinstance(v, dict) else v)
                                 for k, v in kw.items()})
    for name, cases in SINGLE.items():
        for i, kw in enumerate(cases):
            out[f"{name}_{i}_knobs"] = np.array(enc(kw))
            out[f"{name}_{i}"] = run_single(name, kw)

    class Stub:  # the attributes of the model the GenerationMixin method reads
        config = types.SimpleNamespace(is_encoder_decoder=True, max_position_embeddings=None, get_text_config=lambda: None)
        _merge_criteria_processor_list = gu.GenerationMixin._merge_criteria_processor_list
    stub = Stub()

    def processors(knobs, n0, parler=None):
        gc = GenerationConfig(eos_token_id=EOS, pad_token_id=1024, bos_token_id=1025, **knobs)
        gc._eos_token_tensor = torch.tensor([EOS])
        custom = lp.LogitsProcessorList([parler] if parler is not None else [])
        return gu.GenerationMixin._get_logits_processor(stub, generation_config=gc, input_ids_seq_length=n0, encoder_input_ids=None,
                                                        logits_processor=custom, device="cpu", model_kwargs={})

    for ci, (knobs, cols, n0) in enumerate(CHAINS):
        parler = ParlerTTSLogitsProcessor(eos_token_id=EOS, num_codebooks=K, batch_size=R // K, device="cpu")
        procs = processors(knobs, n0, parler=parler)
        out[f"chain{ci}_knobs"] = np.array(enc(knobs))
        out[f"chain{ci}_cols_n0"] = np.array([cols, n0])
        out[f"chain{ci}_order"] = np.array(json.dumps([type(p).__name__ for p in procs]))
        s = scores.clone()
        for p in procs:
            s = p(ids[:, :cols], s)
        out[f"chain{ci}_out"] = s.numpy()
    # 0: no processor, 1: a processor that runs, 2: raised (when built or at its first call; the exception's class is kept)
    status = []
    for kw in VALIDATION:
        try:
            procs = processors(dict(kw, do_sample=False, max_length=T + 1), 1)
            s = scores.clone()
            for p in procs:
                s = p(ids, s)
            status.append([1 if len(procs) else 0, ""])
        except Exception as e:  # noqa: BLE001 -- the class is recorded
            status.append([2, type(e).__name__])
    rec = []
    for kw, st in zip(VALIDATION, status):
        sb = kw.get("sequence_bias")
        knob = dict(kw)
        if isinstance(sb, dict):   # JSON cannot key by tuples: [[key items], value] pairs plus a flag
            knob = dict(sequence_bias_dict=[[[int(t) if isinstance(t, (int, np.integer)) else t for t in (k if isinstance(k, tuple) else [k])],
                                             v, isinstance(k, tuple)] for k, v in sb.items()])
        elif isinstance(sb, list):   # keep whether an entry's ids were a tuple (the list form rejects those)
            knob = dict(sequence_bias_list=[[list(e[0]), e[1], isinstance(e[0], tuple)] for e in sb])
        rec.append([knob, st[0], st[1]])
    out["validation"] = np.array(json.dumps(rec))
    np.savez_compressed(os.path.join(HERE, "logits_ext.npz"), **out)
    print("wrote logits_ext.npz:", sorted(out))


if __name__ == "__main__":
    main()
