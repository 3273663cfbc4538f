"""Writes tests/golden/scoring.npz by executing the reference's own code (run once, with the reference importable):

    PARLER_TTS_REFERENCE=<path to a parler-tts checkout> python tests/golden/make_scoring_golden.py

What is executed: parler_tts shift_tokens_right (:308-323) on labels in training format, then ParlerTTSForCausalLM.forward(
use_cache=False, labels=...) (:1865-1974, loss at :1922-1974) in fp32 at the tiny shape of make_golden.gen_decoder, with a prompt
prefix under a padding mask and a description with masked positions, for loss_reduction "mean" and "sum", with and without
config.codebook_weights.  Saved: the inputs, the decoder input, the logits of the label positions, the loss and the per-codebook
losses of each case.  Import shims: make_golden.import_reference (SURVEY.md section 8c).
"""
from __future__ import annotations
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import ROOT, import_reference  # noqa: E402

WEIGHTS = [1.0, 2.0, 0.5, 3.0]


def training_labels(cfg, lengths, g):
    """Labels [B, T, K] in the delayed training format: codebook k starts k cells late (BOS before it), ends with EOS cells up to
    the delayed end, and -100 right padding for utterances shorter than the longest."""
    K, bos, eos = cfg.num_codebooks, cfg.bos_token_id, cfg.eos_token_id
    T = max(lengths) + K
    labels = torch.full((len(lengths), T, K), -100, dtype=torch.long)
    for b, n in enumerate(lengths):
        codes = torch.randint(0, cfg.codebook_size, (K, n), generator=g)
        for k in range(K):
            row = [bos] * k + codes[k].tolist() + [eos] * (K - k)
            labels[b, :len(row), k] = torch.tensor(row)
    return labels


def gen_scoring(pt):
    from parler_tts import ParlerTTSDecoderConfig, ParlerTTSForCausalLM
    from parler_tts.modeling_parler_tts import shift_tokens_right
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
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    g = torch.Generator().manual_seed(23)
    B, K, P, S = 3, cfg.num_codebooks, 5, 7
    labels = training_labels(cfg, [6, 4, 2], g)
    T = labels.shape[1]
    dec = shift_tokens_right(labels, cfg.pad_token_id, cfg.bos_token_id).transpose(1, 2)   # [B, K, T] (:2820-2823)
    enc = torch.randn(B, S, cfg.hidden_size, generator=g)
    enc_mask = torch.ones(B, S, dtype=torch.long)
    enc_mask[1, :3] = 0
    enc_mask[2, :1] = 0
    enc = enc * enc_mask[..., None]
    prompt = torch.randn(B, P, cfg.hidden_size, generator=g) * 0.5
    pmask = torch.ones(B, P, dtype=torch.long)
    pmask[0, :2] = 0
    out = dict(labels=labels.numpy(), dec=dec.numpy(), enc=enc.numpy(), enc_mask=enc_mask.numpy(), prompt=prompt.numpy(),
               pmask=pmask.numpy(), weights=np.array(WEIGHTS), meta=np.array([B, K, T, P, S]))
    for red in ("mean", "sum"):
        for wname, cw in (("nw", None), ("w", WEIGHTS)):
            m.config.codebook_weights = cw
            with torch.no_grad():
                o = m(input_ids=dec, encoder_hidden_states=enc, encoder_attention_mask=enc_mask, prompt_hidden_states=prompt,
                      prompt_attention_mask=pmask, labels=labels, use_cache=False, loss_reduction=red)
            out[f"{red}_{wname}_loss"] = o.loss.numpy()
            out[f"{red}_{wname}_per_codebook"] = torch.stack(o.per_codebook_losses).numpy()
            out["logits"] = o.logits[:, -T:].numpy()   # [B*K, T, V]
    np.savez_compressed(os.path.join(HERE, "scoring.npz"), **out)


if __name__ == "__main__":
    torch.manual_seed(0)
    gen_scoring(import_reference())
    print("scoring.npz", os.path.getsize(os.path.join(HERE, "scoring.npz")))
