"""Writes tests/golden/prompt_cross.npz by executing the reference's own code (run once, with the reference importable):

    PARLER_TTS_REFERENCE=<path to a parler-tts checkout> python tests/golden/make_prompt_cross_golden.py

What is executed, in fp32 at the tiny shape of make_golden.gen_decoder with config.prompt_cross_attention=True:
  * ParlerTTSForConditionalGeneration._prepare_prompt_kwargs_for_generation (:3099-3130), called on a stand-in `self` that
    carries what the method reads: the embed_prompts table and a real ParlerTTSSinusoidalPositionalEmbedding (:2397-2402);
    once per combination of description mask and prompt mask (both, description only, prompt only, neither);
  * ParlerTTSForCausalLM.forward(use_cache=False, labels=...) (:1865-1974) over the resulting encoder states and mask, with no
    prompt prefix: the logits of every decoder position and the loss.
Saved: the inputs, the concatenated states and mask, the logits and the loss of each case.  Import shims: make_golden.import_reference.
"""
from __future__ import annotations
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import ROOT, import_reference  # noqa: E402
from make_scoring_golden import training_labels  # noqa: E402

# (description mask given, prompt mask given)
CASES = [(True, True), (True, False), (False, True), (False, False)]


def gen_prompt_cross(pt):
    from transformers.modeling_outputs import BaseModelOutput
    from parler_tts import ParlerTTSDecoderConfig, ParlerTTSForCausalLM
    from parler_tts.modeling_parler_tts import (ParlerTTSForConditionalGeneration, ParlerTTSSinusoidalPositionalEmbedding,
                                                shift_tokens_right)
    sys.path.insert(0, ROOT)
    from oracle.config import tiny_cfg
    from oracle.weights import make_decoder_weights
    cfg = tiny_cfg()
    w = make_decoder_weights(cfg, seed=13)
    rc = ParlerTTSDecoderConfig(
        vocab_size=cfg.vocab_size, max_position_embeddings=cfg.max_position_embeddings,
        num_hidden_layers=cfg.num_hidden_layers, ffn_dim=cfg.ffn_dim, num_attention_heads=cfg.num_attention_heads,
        num_key_value_heads=cfg.num_key_value_heads, num_cross_attention_key_value_heads=cfg.num_cross_attention_key_value_heads,
        hidden_size=cfg.hidden_size, num_codebooks=cfg.num_codebooks, pad_token_id=cfg.pad_token_id,
        eos_token_id=cfg.eos_token_id, bos_token_id=cfg.bos_token_id, dropout=0.0,
        rope_embeddings=cfg.rope_embeddings, activation_function=cfg.activation_function)
    rc._attn_implementation = "sdpa"
    m = ParlerTTSForCausalLM(rc).eval()
    sd = {k[len("decoder."):]: v for k, v in w.items() if k.startswith("decoder.")}
    _, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    embed_prompts = torch.nn.Embedding(cfg.text_vocab_size, cfg.hidden_size)
    embed_prompts.weight.data.copy_(w["embed_prompts.weight"])
    stub = types.SimpleNamespace(embed_prompts=embed_prompts, prompt_cross_attention=True, device="cpu",
                                 embed_positions=ParlerTTSSinusoidalPositionalEmbedding(cfg.max_position_embeddings, cfg.hidden_size))

    g = torch.Generator().manual_seed(29)
    B, K, P, S = 3, cfg.num_codebooks, 5, 7
    labels = training_labels(cfg, [6, 4, 3], g)
    T = labels.shape[1]
    dec = shift_tokens_right(labels, cfg.pad_token_id, cfg.bos_token_id).transpose(1, 2)   # [B, K, T] (:2820-2823)
    enc_mask = torch.ones(B, S, dtype=torch.long)
    enc_mask[1, :3] = 0
    enc_mask[2, :1] = 0
    enc = torch.randn(B, S, cfg.hidden_size, generator=g) * enc_mask[..., None]   # multiplied by its mask (:3092-3093)
    prompt_ids = torch.randint(0, cfg.text_vocab_size, (B, P), generator=g)
    pmask = torch.ones(B, P, dtype=torch.long)
    pmask[0, :2] = 0
    pmask[2, :1] = 0
    out = dict(labels=labels.numpy(), dec=dec.numpy(), enc=enc.numpy(), enc_mask=enc_mask.numpy(), prompt_ids=prompt_ids.numpy(),
               pmask=pmask.numpy(), meta=np.array([B, K, T, P, S]), cases=np.array(CASES, dtype=np.int64))
    for ci, (use_em, use_pm) in enumerate(CASES):
        mk = {"encoder_outputs": BaseModelOutput(last_hidden_state=enc.clone()), "attention_mask": enc_mask.clone() if use_em else None,
              "prompt_attention_mask": pmask.clone() if use_pm else None}
        with torch.no_grad():
            mk = ParlerTTSForConditionalGeneration._prepare_prompt_kwargs_for_generation(stub, prompt_ids, mk)
        assert mk["prompt_hidden_states"] is None and mk["prompt_attention_mask"] is None
        states, mask = mk["encoder_outputs"].last_hidden_state, mk["attention_mask"]
        with torch.no_grad():
            o = m(input_ids=dec, encoder_hidden_states=states, encoder_attention_mask=mask, labels=labels, use_cache=False)
        out[f"c{ci}_states"] = states.numpy()
        out[f"c{ci}_has_mask"] = np.array(int(mask is not None))
        out[f"c{ci}_mask"] = (mask if mask is not None else torch.zeros(0, dtype=torch.long)).numpy()
        out[f"c{ci}_logits"] = o.logits.numpy()   # [B*K, T, V]
        out[f"c{ci}_loss"] = o.loss.numpy()
    np.savez_compressed(os.path.join(HERE, "prompt_cross.npz"), **out)


if __name__ == "__main__":
    torch.manual_seed(0)
    gen_prompt_cross(import_reference())
    print("prompt_cross.npz", os.path.getsize(os.path.join(HERE, "prompt_cross.npz")))
