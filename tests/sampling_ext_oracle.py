"""CPU restatement of the processors generate() adds through ptts_sampling_ext (test infrastructure only).

  NoRepeatNGramLogitsProcessor          transformers `generation/logits_process.py` (_get_ngrams / _calc_banned_ngram_tokens)
  MinP / Typical / Epsilon / Eta        the warpers of the same file, min_tokens_to_keep = 1
  MinLength                             folded into MinNewTokens: min_new_tokens = max(0, min_length - n0) unless min_new_tokens
                                        is given (`_prepare_generated_length`)
  processor order                       [NoRepeatNGram, MinLength / MinNewTokens, ParlerTTS (custom), Temperature, TopK, TopP,
                                         MinP, Typical, Epsilon, Eta] (`_get_logits_processor`)
PINNED bit-exact against those classes by tests/golden/sampling_ext.npz (make_sampling_ext_golden.py).  Built on the oracle's
own pieces (oracle/sampling.py, tests/continuation_oracle.py).
"""
from __future__ import annotations
import math

import numpy as np
import torch

from oracle.delay_pattern import apply_delay_pattern_mask, build_delay_pattern_mask
from oracle.sampling import ParlerLogitsProcessorOracle, min_new_tokens, temperature, top_k, top_p
from tests.continuation_oracle import bos_led, generated_length


def no_repeat_ngram(ids: np.ndarray, scores: np.ndarray, n: int) -> np.ndarray:
    """ids [R, cur_len]: the next id of every earlier n-gram whose first n - 1 ids equal the row's last n - 1 goes to -inf."""
    R, cur = ids.shape
    out = scores.copy()
    if n <= 0 or cur + 1 < n:
        return out
    for r in range(R):
        row = [int(t) for t in ids[r]]
        tail = tuple(row[cur - n + 1:])
        for i in range(cur - n + 1):
            if tuple(row[i:i + n - 1]) == tail:
                out[r, row[i + n - 1]] = -math.inf
    return out


def min_p(scores: np.ndarray, p: float) -> np.ndarray:
    t = torch.from_numpy(scores)
    probs = t.softmax(-1)
    rm = probs < p * probs.amax(-1, keepdim=True)
    rm.scatter_(-1, torch.topk(probs, 1, dim=-1).indices, False)
    return t.masked_fill(rm, -math.inf).numpy()


def typical(scores: np.ndarray, mass: float) -> np.ndarray:
    t = torch.from_numpy(scores)
    nl = torch.nn.functional.log_softmax(t, dim=-1)
    ent = -(nl * torch.exp(nl)).nansum(-1, keepdim=True)
    shifted = torch.abs(-nl - ent)
    ss, si = torch.sort(shifted, descending=False)
    cum = t.gather(-1, si).softmax(-1).cumsum(-1)
    last = (cum < mass).sum(1).clamp(max=ss.shape[-1] - 1)
    rm = ss > ss.gather(1, last.view(-1, 1))
    rm[..., :1] = False
    return t.masked_fill(rm.scatter(1, si, rm), -math.inf).numpy()


def entropy(scores: np.ndarray) -> np.ndarray:
    return torch.distributions.Categorical(logits=torch.from_numpy(scores)).entropy().numpy()


def epsilon(scores: np.ndarray, eps: float) -> np.ndarray:
    t = torch.from_numpy(scores)
    rm = (t.softmax(-1) < eps) & (t < torch.topk(t, 1)[0][..., -1, None])
    return t.masked_fill(rm, -math.inf).numpy()


def eta_threshold(scores: np.ndarray, eps: float) -> np.ndarray:
    e = torch.tensor(eps)
    ent = torch.distributions.Categorical(logits=torch.from_numpy(scores)).entropy()
    return torch.min(e, torch.sqrt(e) * torch.exp(-ent))[..., None].numpy()


def eta(scores: np.ndarray, eps: float) -> np.ndarray:
    t = torch.from_numpy(scores)
    rm = (t.softmax(-1) < torch.from_numpy(eta_threshold(scores, eps))) & (t < torch.topk(t, 1)[0][..., -1, None])
    return t.masked_fill(rm, -math.inf).numpy()


def folded_min_new_tokens(min_length, min_new, n0: int) -> int:
    if min_new is not None:
        return int(min_new)
    return max(0, int(min_length) - n0) if (min_length or 0) > 0 else 0


WARPERS = (("min_p", min_p, None), ("typical_p", typical, 1.0), ("epsilon_cutoff", epsilon, None), ("eta_cutoff", eta, None))


def warper_on(gen: dict, name: str) -> bool:
    v = gen.get(name)
    if name == "min_p":
        return v is not None
    if name == "typical_p":
        return v is not None and v < 1.0
    return v is not None and 0.0 < v < 1.0


def process_scores(scores: np.ndarray, raw_ids: np.ndarray, parler: ParlerLogitsProcessorOracle, gen: dict, n0: int = 1,
                   stages: list | None = None) -> np.ndarray:
    """One step's chain on fp32 scores [B*K, V]; raw_ids = the un-masked history (Q10).  gen: the generate() knobs.
    stages, if given, collects (name, scores after the stage) for every warper after top-p."""
    s = scores.astype(np.float32).copy()
    s = no_repeat_ngram(raw_ids, s, int(gen.get("no_repeat_ngram_size") or 0))
    mnt = folded_min_new_tokens(gen.get("min_length"), gen.get("min_new_tokens"), n0)
    if mnt > 0:
        s = min_new_tokens(s, raw_ids.shape[1], n0, mnt, parler.eos)
    s = parler(raw_ids, s)
    if gen.get("do_sample", False):
        if gen.get("temperature", 1.0) != 1.0:
            s = temperature(s, gen["temperature"])
        if gen.get("top_k", 0):
            s = top_k(s, gen["top_k"])
        if gen.get("top_p", 1.0) < 1.0:
            s = top_p(s, gen["top_p"])
        for name, fn, _ in WARPERS:
            if warper_on(gen, name):
                if stages is not None:
                    stages.append((name, s.copy()))
                s = fn(s, gen[name])
    return s


def generate_tokens(dec, cfg, enc_hidden, enc_mask, prompt_hidden, prompt_mask, gen: dict, decoder_input_ids=None, pick=None):
    """tests.continuation_oracle.generate_tokens with this module's chain; greedy unless `pick(step, scores)` draws.
    Returns dict(raw_ids [B*K, n], input_ids, max_length, n0, scores list)."""
    B = enc_hidden.shape[0]
    K, bos, pad, eos = cfg.num_codebooks, cfg.bos_token_id, cfg.pad_token_id, cfg.eos_token_id
    input_ids = np.full((B * K, 1), bos, dtype=np.int64) if decoder_input_ids is None else bos_led(decoder_input_ids, K, bos)
    n0 = input_ids.shape[1]
    L = generated_length(n0, gen.get("max_new_tokens"), gen.get("max_length", 0))
    ids, delay_mask = build_delay_pattern_mask(input_ids, bos, pad, L, K)
    parler = ParlerLogitsProcessorOracle(eos, K, B)
    unfinished = np.ones(B * K, dtype=np.int64)
    all_scores = []
    step = 0
    while True:
        model_in = apply_delay_pattern_mask(ids, delay_mask)
        if step == 0:
            logits = dec.prefill(torch.from_numpy(model_in), enc_hidden, enc_mask, prompt_hidden, prompt_mask)
        else:
            logits = dec.step(torch.from_numpy(model_in[:, -1:]))
        s = process_scores(logits[:, -1, :].float().numpy(), ids, parler, gen, n0)
        all_scores.append(s.copy())
        nxt = pick(step, s) if pick is not None else s.argmax(-1)
        nxt = nxt * unfinished + pad * (1 - unfinished)
        ids = np.concatenate([ids, nxt[:, None]], axis=1)
        done = (ids[:, -1] == eos) | (ids.shape[1] >= L)
        unfinished = unfinished & ~done
        step += 1
        if unfinished.max() == 0:
            break
    return dict(raw_ids=ids, input_ids=input_ids, max_length=L, n0=n0, scores=all_scores)
