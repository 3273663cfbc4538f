"""CPU restatement of the processors generate() adds through ptts_logits_ext (test infrastructure only).

  SequenceBiasLogitsProcessor             transformers `generation/logits_process.py`: bias = 0 + the single-id biases, then each
                                          multi-id sequence whose prefix ends the history adds its bias to its last id, in dict
                                          order (sequences longer than the history are skipped); scores + bias, all in fp32
  SuppressTokens / SuppressTokensAtBegin  -inf at the listed ids (out-of-vocabulary ids ignored); the second only at
                                          cur_len == begin_index
  ExponentialDecayLengthPenalty           regulation_start = start + n0; past it scores + penalties with
                                          penalties[eos] = |scores[eos]| * fp32(pow(factor, cur_len - regulation_start) - 1)
  ForcedBOS / ForcedEOS                   the whole row -inf but the forced id at 0, at cur_len == 1 / cur_len == max_length - 1
  InfNanRemove                            NaN -> 0, +-inf -> +-finfo(float32).max
  LogitNormalization                      log_softmax, after every other processor and warper
  order                                   [SequenceBias, NoRepeatNGram, MinLength / MinNewTokens, ForcedBOS, ForcedEOS, InfNan,
                                           ExponentialDecay, Suppress, SuppressAtBegin, ParlerTTS (custom), Temperature ..
                                           Eta, LogitNormalization] (`_get_logits_processor`)
PINNED bit-exact against those classes by tests/golden/logits_ext.npz (make_logits_ext_golden.py).  Built on
tests/sampling_ext_oracle.py and the oracle's own pieces.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.sampling import ParlerLogitsProcessorOracle, min_new_tokens, temperature, top_k, top_p
from tests import sampling_ext_oracle as so

F32_MAX = np.float32(np.finfo(np.float32).max)


def seq_bias_dict(sb) -> dict:
    """Either format -> {tuple(ids): float} in the given order (the list form's later duplicates overwrite in place)."""
    if isinstance(sb, dict):
        return {tuple(int(t) for t in k): float(v) for k, v in sb.items()}
    return {tuple(int(t) for t in e[0]): float(e[1]) for e in sb}


def sequence_bias(ids: np.ndarray, scores: np.ndarray, sb) -> np.ndarray:
    sb = seq_bias_dict(sb)
    R, V = scores.shape
    bias = np.zeros((R, V), dtype=np.float32)
    l1 = np.zeros(V, dtype=np.float32)
    for k, b in sb.items():
        if len(k) == 1:
            l1[k[0]] = np.float32(b)
    bias = bias + l1
    cur = ids.shape[1]
    for k, b in sb.items():
        if len(k) == 1 or len(k) > cur:
            continue
        match = (ids[:, cur - len(k) + 1:] == np.array(k[:-1])[None, :]).all(1)
        bias[:, k[-1]] = bias[:, k[-1]] + np.where(match, np.float32(b), np.float32(0.0))
    return (scores.astype(np.float32) + bias).astype(np.float32)


def suppress(scores: np.ndarray, tokens) -> np.ndarray:
    out = scores.copy()
    for t in tokens:
        if 0 <= t < scores.shape[1]:
            out[:, t] = -np.inf
    return out


def begin_suppress(ids: np.ndarray, scores: np.ndarray, tokens, begin_index: int) -> np.ndarray:
    return suppress(scores, tokens) if ids.shape[1] == begin_index else scores.copy()


def begin_index(n0: int, forced_bos) -> int:
    return n0 + (1 if n0 == 1 and forced_bos is not None else 0)


def decay_multiplier(start: int, factor: float, n0: int, cur_len: int) -> np.float32:
    """fp32(pow(factor, cur_len - regulation_start) - 1), the scalar transformers multiplies the fp32 EOS score with."""
    return np.float32(pow(factor, cur_len - (start + n0)) - 1)


def decay_table(start: int, factor: float, n0: int, max_length: int) -> np.ndarray:
    t = np.zeros(max_length, dtype=np.float32)
    for c in range(start + n0 + 1, max_length):
        t[c] = decay_multiplier(start, factor, n0, c)
    return t


def exponential_decay(ids: np.ndarray, scores: np.ndarray, start: int, factor: float, n0: int, eos: int) -> np.ndarray:
    cur = ids.shape[1]
    if cur <= start + n0:
        return scores.copy()
    pen = np.zeros_like(scores)
    with np.errstate(invalid="ignore", over="ignore"):
        pen[:, eos] = np.abs(scores[:, eos]) * decay_multiplier(start, factor, n0, cur)
        return (scores + pen).astype(np.float32)


def forced(scores: np.ndarray, token: int) -> np.ndarray:
    out = np.full_like(scores, -np.inf)
    out[:, token] = 0.0
    return out


def infnan(scores: np.ndarray) -> np.ndarray:
    out = np.where(np.isnan(scores), np.float32(0.0), scores)
    out = np.where(scores == np.inf, F32_MAX, out)
    return np.where(scores == -np.inf, -F32_MAX, out).astype(np.float32)


def log_softmax(scores: np.ndarray) -> np.ndarray:
    return torch.from_numpy(scores).log_softmax(-1).numpy()


def process_scores(scores: np.ndarray, raw_ids: np.ndarray, parler: ParlerLogitsProcessorOracle, gen: dict, n0: int = 1,
                   max_length: int | None = None) -> np.ndarray:
    """One step's chain on fp32 scores [B*K, V]; raw_ids = the un-masked history [B*K, cur_len].  gen: the generate() knobs
    (those of sampling_ext_oracle.process_scores plus this module's); max_length: the resolved max_length (forced EOS)."""
    s = scores.astype(np.float32).copy()
    cur, eos = raw_ids.shape[1], parler.eos
    if gen.get("sequence_bias") is not None:
        s = sequence_bias(raw_ids, s, gen["sequence_bias"])
    s = so.no_repeat_ngram(raw_ids, s, int(gen.get("no_repeat_ngram_size") or 0))
    mnt = so.folded_min_new_tokens(gen.get("min_length"), gen.get("min_new_tokens"), n0)
    if mnt > 0:
        s = min_new_tokens(s, cur, n0, mnt, eos)
    if gen.get("forced_bos_token_id") is not None and cur == 1:
        s = forced(s, gen["forced_bos_token_id"])
    if gen.get("forced_eos_token_id") is not None and cur == max_length - 1:
        s = forced(s, gen["forced_eos_token_id"])
    if gen.get("remove_invalid_values") is True:
        s = infnan(s)
    if gen.get("exponential_decay_length_penalty") is not None:
        start, factor = gen["exponential_decay_length_penalty"]
        s = exponential_decay(raw_ids, s, start, factor, n0, eos)
    if gen.get("suppress_tokens") is not None:
        s = suppress(s, gen["suppress_tokens"])
    if gen.get("begin_suppress_tokens") is not None:
        s = begin_suppress(raw_ids, s, gen["begin_suppress_tokens"], begin_index(n0, gen.get("forced_bos_token_id")))
    s = parler(raw_ids, s)
    if gen.get("do_sample", False):
        if gen.get("temperature", 1.0) != 1.0:
            s = temperature(s, gen["temperature"])
        if gen.get("top_k", 0):
            s = top_k(s, gen["top_k"])
        if gen.get("top_p", 1.0) < 1.0:
            s = top_p(s, gen["top_p"])
        for name, fn, _ in so.WARPERS:
            if so.warper_on(gen, name):
                s = fn(s, gen[name])
    if gen.get("renormalize_logits") is True:
        s = log_softmax(s)
    return s


def pre_normalization(gen: dict) -> dict:
    """The same knobs without LogitNormalization: the scores greedy's argmax and the draw use."""
    return {k: v for k, v in gen.items() if k != "renormalize_logits"}


def generate_tokens(dec, cfg, enc_hidden, enc_mask, prompt_hidden, prompt_mask, gen: dict, decoder_input_ids=None):
    """Greedy free-running loop of sampling_ext_oracle.generate_tokens with this module's chain (argmax before LogitNormalization).
    Returns dict(raw_ids [B*K, n], input_ids, max_length, n0, scores list of the pre-normalization rows)."""
    from oracle.delay_pattern import apply_delay_pattern_mask, build_delay_pattern_mask
    from tests.continuation_oracle import bos_led, generated_length
    B = enc_hidden.shape[0]
    K, bos, pad, eos = cfg.num_codebooks, cfg.bos_token_id, cfg.pad_token_id, cfg.eos_token_id
    input_ids = np.full((B * K, 1), bos, dtype=np.int64) if decoder_input_ids is None else bos_led(decoder_input_ids, K, bos)
    n0 = input_ids.shape[1]
    L = generated_length(n0, gen.get("max_new_tokens"), gen.get("max_length", 0))
    ids, delay_mask = build_delay_pattern_mask(input_ids, bos, pad, L, K)
    parler = ParlerLogitsProcessorOracle(eos, K, B)
    unfinished = np.ones(B * K, dtype=np.int64)
    all_scores, step = [], 0
    g = pre_normalization(gen)
    while True:
        model_in = apply_delay_pattern_mask(ids, delay_mask)
        if step == 0:
            logits = dec.prefill(torch.from_numpy(model_in), enc_hidden, enc_mask, prompt_hidden, prompt_mask)
        else:
            logits = dec.step(torch.from_numpy(model_in[:, -1:]))
        s = process_scores(logits[:, -1, :].float().numpy(), ids, parler, g, n0, L)
        all_scores.append(s.copy())
        nxt = s.argmax(-1)
        nxt = nxt * unfinished + pad * (1 - unfinished)
        ids = np.concatenate([ids, nxt[:, None]], axis=1)
        unfinished = unfinished & ~((ids[:, -1] == eos) | (ids.shape[1] >= L))
        step += 1
        if unfinished.max() == 0:
            break
    return dict(raw_ids=ids, input_ids=input_ids, max_length=L, n0=n0, scores=all_scores)

