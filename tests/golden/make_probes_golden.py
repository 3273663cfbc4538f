"""Writes tests/golden/probes.npz by executing the reference's own code (run once, with the reference importable):

    PARLER_TTS_REFERENCE=<path to a parler-tts checkout> python tests/golden/make_probes_golden.py

What is executed: ParlerTTSForCausalLM.forward(use_cache=False, output_attentions=True, output_hidden_states=True) (:1865-1974)
with the EAGER attention (ParlerTTSAttention, :494-584) in fp32 at the tiny shape of make_golden.gen_decoder, with a prompt
prefix under a padding mask and a description with masked positions, in three cases: sinusoidal positions with one K/V head per
query head, RoPE with one K/V head per query head, and RoPE with grouped-query attention (two query heads per K/V head, self and
cross).  Saved per case: the inputs, the decoder input ids, the L self-attention and cross-attention weight tensors and the L + 1
hidden-state tensors in the reference's order.  Import shims: make_golden.import_reference (SURVEY.md section 8c).
"""
from __future__ import annotations
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import ROOT, import_reference  # noqa: E402

# name -> (tiny_cfg overrides, weight seed)
CASES = {
    "sin": (dict(), 31),
    "rope": (dict(rope_embeddings=True), 32),
    "rope_gqa": (dict(rope_embeddings=True, hidden_size=256, num_attention_heads=4, num_key_value_heads=2,
                      num_cross_attention_key_value_heads=2), 33),
}


def gen_probes(pt):
    from parler_tts import ParlerTTSDecoderConfig, ParlerTTSForCausalLM
    sys.path.insert(0, ROOT)
    from oracle.config import tiny_cfg
    from oracle.weights import make_decoder_weights
    out = {}
    for name, (over, seed) in CASES.items():
        cfg = tiny_cfg(**over)
        w = make_decoder_weights(cfg, seed=seed)
        rc = ParlerTTSDecoderConfig(
            vocab_size=cfg.vocab_size, max_position_embeddings=cfg.max_position_embeddings,
            num_hidden_layers=cfg.num_hidden_layers, ffn_dim=cfg.ffn_dim, num_attention_heads=cfg.num_attention_heads,
            num_key_value_heads=cfg.num_key_value_heads, num_cross_attention_key_value_heads=cfg.num_cross_attention_key_value_heads,
            hidden_size=cfg.hidden_size, num_codebooks=cfg.num_codebooks, pad_token_id=cfg.pad_token_id,
            eos_token_id=cfg.eos_token_id, bos_token_id=cfg.bos_token_id, dropout=0.0,
            rope_embeddings=cfg.rope_embeddings, activation_function=cfg.activation_function)
        rc._attn_implementation = "eager"
        m = ParlerTTSForCausalLM(rc).eval()
        sd = {k[len("decoder."):]: v for k, v in w.items() if k.startswith("decoder.")}
        missing, unexpected = m.load_state_dict(sd, strict=False)
        assert not unexpected, unexpected
        g = torch.Generator().manual_seed(seed)
        B, K, P, S, T = 2, cfg.num_codebooks, 5, 7, 6
        dec = torch.randint(0, cfg.codebook_size, (B, K, T), generator=g)
        dec[:, :, 0] = cfg.bos_token_id
        enc = torch.randn(B, S, cfg.hidden_size, generator=g)
        enc_mask = torch.ones(B, S, dtype=torch.long)
        enc_mask[1, :3] = 0
        enc = enc * enc_mask[..., None]
        prompt = torch.randn(B, P, cfg.hidden_size, generator=g) * 0.5
        pmask = torch.ones(B, P, dtype=torch.long)
        pmask[0, :2] = 0
        with torch.no_grad():
            o = m(input_ids=dec.reshape(B * K, T), encoder_hidden_states=enc, encoder_attention_mask=enc_mask, prompt_hidden_states=prompt,
                  prompt_attention_mask=pmask, use_cache=False, output_attentions=True, output_hidden_states=True)
        L = cfg.num_hidden_layers
        assert len(o.attentions) == L and len(o.cross_attentions) == L and len(o.hidden_states) == L + 1
        out[f"{name}_meta"] = np.array([B, K, P, S, T, seed])
        out[f"{name}_dec"] = dec.reshape(B * K, T).numpy()
        out[f"{name}_enc"], out[f"{name}_enc_mask"] = enc.numpy(), enc_mask.numpy()
        out[f"{name}_prompt"], out[f"{name}_pmask"] = prompt.numpy(), pmask.numpy()
        out[f"{name}_self"] = torch.stack(o.attentions).numpy()            # [L, B, heads, P+T, P+T]
        out[f"{name}_cross"] = torch.stack(o.cross_attentions).numpy()     # [L, B, heads, P+T, S]
        out[f"{name}_hidden"] = torch.stack(o.hidden_states).numpy()       # [L+1, B, P+T, H]
    np.savez_compressed(os.path.join(HERE, "probes.npz"), **out)


if __name__ == "__main__":
    torch.manual_seed(0)
    gen_probes(import_reference())
    print("probes.npz", os.path.getsize(os.path.join(HERE, "probes.npz")))
