"""CPU restatement of generate() continuing from audio codes (test infrastructure only).

  BOS column prepend          modeling_parler_tts.py:3012-3024 (_prepare_decoder_input_ids_for_generation)
  generated length            transformers `_prepare_generated_length`: max_new_tokens + n0, else max_length is the total
  delay pattern of the input  :3523 (build_delay_pattern_mask over the whole BOS-led input)
  step 0                      [prompt_hidden_states || embed-sum of the n0 delayed columns] (:3033-3044), one forward
  MinNewTokens                prompt_length_to_skip = n0
  next-input override         prepare_inputs_for_generation applies the pattern mask (:2909), the raw token stays in the history
  de-delay                    :3586-3597 with both masks built from the BOS-led input
Built on the oracle's own pieces (oracle/delay_pattern.py, oracle/sampling.py); tests/golden/continuation.npz pins the integer
parts against the reference's code.
"""
from __future__ import annotations
import numpy as np
import torch

from oracle.delay_pattern import apply_delay_pattern_mask, build_delay_pattern_mask
from oracle.sampling import ParlerLogitsProcessorOracle, min_new_tokens, softmax_rows, temperature, top_k, top_p


def bos_led(decoder_input_ids: np.ndarray, num_codebooks: int, start: int) -> np.ndarray:
    """:3012-3024 -- reshape(-1, K, N) accepted, BOS column prepended unless every row already starts with it."""
    ids = np.asarray(decoder_input_ids, dtype=np.int64)
    ids = ids.reshape(-1, ids.shape[-1])
    if (ids[:, 0] != start).all():
        ids = np.concatenate([np.full((ids.shape[0], 1), start, dtype=np.int64), ids], axis=1)
    return ids


def generated_length(n0: int, max_new_tokens: int | None, max_length: int) -> int:
    return int(max_new_tokens) + n0 if max_new_tokens is not None else int(max_length)


def codes_from_raw(raw_ids: np.ndarray, input_ids: np.ndarray, cfg, B: int, max_length: int) -> np.ndarray:
    """:3586-3597: apply the stashed mask (built at max_length), rebuild at the output's length, keep the free cells."""
    K, bos, pad = cfg.num_codebooks, cfg.bos_token_id, cfg.pad_token_id
    _, stashed = build_delay_pattern_mask(input_ids, bos, pad, max_length, K)
    out = apply_delay_pattern_mask(raw_ids, stashed)
    _, mask = build_delay_pattern_mask(input_ids, bos, pad, out.shape[1], K)
    keep = (mask != bos) & (mask != pad)
    return out[keep].reshape(B, K, -1)


def generate_tokens(dec, cfg, enc_hidden, enc_mask, prompt_hidden, prompt_mask, gen: dict, decoder_input_ids=None,
                    collect_logits=False):
    """oracle.sampling.generate_tokens with `decoder_input_ids` (greedy or multinomial).

    gen: max_length (total, prefix included) or max_new_tokens, do_sample, temperature, top_k, top_p, min_new_tokens.
    Returns dict(raw_ids [B*K, n], input_ids (BOS-led), delay_mask, max_length, n0, logits list)."""
    B = enc_hidden.shape[0]
    K, bos, pad, eos = cfg.num_codebooks, cfg.bos_token_id, cfg.pad_token_id, cfg.eos_token_id
    if decoder_input_ids is None:
        input_ids = np.full((B * K, 1), bos, dtype=np.int64)
    else:
        input_ids = bos_led(decoder_input_ids, K, bos)
    n0 = input_ids.shape[1]
    L = generated_length(n0, gen.get("max_new_tokens"), gen.get("max_length", 0))
    ids, delay_mask = build_delay_pattern_mask(input_ids, bos, pad, L, K)
    parler = ParlerLogitsProcessorOracle(eos, K, B)
    unfinished = np.ones(B * K, dtype=np.int64)
    all_logits = []
    step = 0
    while True:
        model_in = apply_delay_pattern_mask(ids, delay_mask)
        if step == 0:
            logits = dec.prefill(torch.from_numpy(model_in), enc_hidden, enc_mask, prompt_hidden, prompt_mask)
        else:
            logits = dec.step(torch.from_numpy(model_in[:, -1:]))
        nl = logits[:, -1, :].float().numpy()
        s = nl.astype(np.float32).copy()
        if gen.get("min_new_tokens", 0) > 0:
            s = min_new_tokens(s, ids.shape[1], n0, gen["min_new_tokens"], eos)
        s = parler(ids, s)
        if gen.get("do_sample", False):
            if gen.get("temperature", 1.0) != 1.0:
                s = temperature(s, gen["temperature"])
            if gen.get("top_k", 0):
                s = top_k(s, gen["top_k"])
            if gen.get("top_p", 1.0) < 1.0:
                s = top_p(s, gen["top_p"])
            nxt = torch.multinomial(torch.from_numpy(softmax_rows(s)), 1).squeeze(1).numpy()
        else:
            nxt = s.argmax(-1)
        if collect_logits:
            all_logits.append(nl.copy())
        nxt = nxt * unfinished + pad * (1 - unfinished)
        ids = np.concatenate([ids, nxt[:, None]], axis=1)
        done = (ids[:, -1] == eos) | (ids.shape[1] >= L)
        unfinished = unfinished & ~done
        step += 1
        if unfinished.max() == 0:
            break
    return dict(raw_ids=ids, input_ids=input_ids, delay_mask=delay_mask, max_length=L, n0=n0, logits=all_logits)
