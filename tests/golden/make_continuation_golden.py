"""Writes tests/golden/continuation.npz by executing the reference's own code (run once, with the reference importable):

    PARLER_TTS_REFERENCE=<path to a parler-tts checkout> python tests/golden/make_continuation_golden.py

Per case (B, K, N, leading BOS or not, max_new_tokens, max_length):
  * input_ids   -- ParlerTTSForConditionalGeneration._prepare_decoder_input_ids_for_generation (:2988-3046), called on a stand-in
                   `self` that carries only what the method reads (prompt_cross_attention=True skips the embedding of step 0);
  * max_length  -- transformers' GenerationMixin._prepare_generated_length with input_ids_length = n0;
  * delayed / mask -- parler_tts build_delay_pattern_mask(input_ids, bos, pad, max_length) (:214-276);
  * codes       -- the generate() tail (:3586-3597) on a random full history, with the reference's apply/build functions.
Import shims: make_golden.import_reference (SURVEY.md section 8c).
"""
from __future__ import annotations
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import import_reference  # noqa: E402

BOS, PAD = 65, 64
# (B, K, N, with_bos, max_new_tokens, max_length)
CASES = [(1, 4, 5, False, 7, None), (2, 4, 6, True, 5, None), (3, 9, 12, False, None, 40), (2, 9, 1, False, 20, None),
         (1, 4, 3, False, None, 6), (2, 4, 2, True, None, 5), (2, 3, 7, False, 4, None), (1, 9, 30, True, None, 45)]


def gen_continuation(pt):
    from transformers import GenerationConfig
    from transformers.generation.utils import GenerationMixin
    from parler_tts.modeling_parler_tts import ParlerTTSForConditionalGeneration, build_delay_pattern_mask, apply_delay_pattern_mask
    out = {}
    g = torch.Generator().manual_seed(17)
    for ci, (B, K, N, with_bos, mnt, ml) in enumerate(CASES):
        codes = torch.randint(0, 64, (B * K, N), generator=g)
        if with_bos:
            codes[:, 0] = BOS
        stub = types.SimpleNamespace(decoder=types.SimpleNamespace(num_codebooks=K), prompt_cross_attention=True, device="cpu",
                                     _get_decoder_start_token_id=lambda start, bos: start)
        input_ids, _ = ParlerTTSForConditionalGeneration._prepare_decoder_input_ids_for_generation(
            stub, batch_size=B, model_input_name="input_ids", model_kwargs={"decoder_input_ids": codes.clone()},
            decoder_start_token_id=torch.tensor(BOS), bos_token_id=torch.tensor(BOS), device="cpu")
        n0 = input_ids.shape[-1]
        gc = GenerationConfig(max_length=ml if ml is not None else 2580, max_new_tokens=mnt)
        lstub = types.SimpleNamespace(config=types.SimpleNamespace(is_encoder_decoder=True, max_position_embeddings=4096))
        gc = GenerationMixin._prepare_generated_length(lstub, gc, has_default_max_length=ml is None, has_default_min_length=True,
                                                       model_input_name="input_ids", input_ids_length=n0,
                                                       inputs_tensor=torch.zeros(B, 3, dtype=torch.long))
        L = int(gc.max_length)
        delayed, mask = build_delay_pattern_mask(input_ids, bos_token_id=BOS, pad_token_id=PAD, max_length=L, num_codebooks=K)
        # a full history: the delayed input, then random tokens up to max_length (the generate() tail at :3586-3597)
        full = torch.cat([delayed, torch.randint(0, 64, (B * K, L - delayed.shape[1]), generator=g)], dim=1)
        applied = apply_delay_pattern_mask(full, mask)
        _, m2 = build_delay_pattern_mask(input_ids, bos_token_id=BOS, pad_token_id=PAD, max_length=applied.shape[1], num_codebooks=K)
        keep = (m2 != BOS) & (m2 != PAD)
        frames = applied[keep].reshape(B, K, -1)
        out[f"c{ci}_meta"] = np.array([B, K, N, int(with_bos), -1 if mnt is None else mnt, -1 if ml is None else ml])
        out[f"c{ci}_codes"] = codes.numpy()
        out[f"c{ci}_input_ids"] = input_ids.numpy()
        out[f"c{ci}_max_length"] = np.array(L)
        out[f"c{ci}_delayed"] = delayed.numpy()
        out[f"c{ci}_mask"] = mask.numpy()
        out[f"c{ci}_full"] = full.numpy()
        out[f"c{ci}_frames"] = frames.numpy()
    out["n"] = np.array(len(CASES))
    out["tokens"] = np.array([BOS, PAD])
    np.savez_compressed(os.path.join(HERE, "continuation.npz"), **out)


if __name__ == "__main__":
    torch.manual_seed(0)
    gen_continuation(import_reference())
    print("continuation.npz", os.path.getsize(os.path.join(HERE, "continuation.npz")))
