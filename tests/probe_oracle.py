"""CPU oracle of output_attentions / output_hidden_states (test infrastructure only).

ProbeOracleDecoder is oracle.decoder.OracleDecoder with every call also recording what the reference returns with
output_attentions=True / output_hidden_states=True:
  * the attention weights by its EAGER attention (ParlerTTSAttention.forward, modeling_parler_tts.py:494-584), which is the path
    it takes when asked for them: q = q_proj(x) * scaling, RoPE, scores = q @ k^T in the model dtype plus the additive mask
    (finfo.min where a key is padded or in the future), softmax computed in fp32 and rounded to the model dtype;
  * the hidden states in ParlerTTSDecoder.forward's order (:1571-1636): the embeddings (plus positions), the outputs of layers
    0 .. L-2, then the final LayerNorm of the last layer's output.
The tokens and logits stay those of OracleDecoder (SDPA).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.decoder import OracleDecoder


def eager_weights(qs, ks, mask_bool, dtype):
    """qs [B, nh, q, hd] (rotated, unscaled), ks [B, nh, T, hd] (repeated to nh heads), mask_bool [B, 1|nh, q, T] True = masked
    -> [B, nh, q, T] in dtype.  scaling = hd ** -0.5 (1/8 for the decoder's head_dim 64)."""
    q = (qs.to(dtype) * qs.shape[-1] ** -0.5).to(dtype)
    s = torch.matmul(q, ks.to(dtype).transpose(2, 3))
    mn = torch.finfo(dtype).min
    s = s + torch.where(mask_bool, torch.tensor(mn, dtype=dtype), torch.tensor(0, dtype=dtype))
    return F.softmax(s.float(), dim=-1).to(dtype)


class ProbeOracleDecoder(OracleDecoder):
    _enc_mask = None

    def reset(self):
        super().reset()
        self.calls = []   # per forward(): dict(self=[L x [B,nh,q,T]], cross=[L x [B,nh,q,S]], hidden=[L+1 x [B,q,H]])

    def _attn(self, layer, x, cross, cos, sin, mask, past, enc=None):
        out = super()._attn(layer, x, cross, cos, sin, mask, past, enc)
        B, q, _ = x.shape
        p = f"layers.{layer}." + ("encoder_attn." if cross else "self_attn.")
        qs = F.linear(x, self._p(p + "q_proj.weight")).view(B, q, self.nh, self.hd).transpose(1, 2).contiguous()
        if self.cfg.rope_embeddings:
            qs = self._apply_rope(qs, cos, sin)
        ks = self.ck[layer] if cross else self.k_cache[layer]
        nkv = ks.shape[1]
        rep = self.nh // nkv
        ks = ks[:, :, None].expand(B, nkv, rep, ks.shape[2], self.hd).reshape(B, self.nh, -1, self.hd)
        T = ks.shape[2]
        if cross:
            m = torch.zeros(B, 1, q, T, dtype=torch.bool)
            if self._enc_mask is not None:
                m = m | (self._enc_mask[:, None, None, :] == 0)
        else:
            pos = torch.arange(past, past + q)[:, None]
            m = (torch.arange(T)[None, :] > pos)[None, None].expand(B, 1, q, T).clone()
            if self.prompt_mask is not None:
                P = self.prompt_mask.shape[1]
                pad = torch.zeros(B, T, dtype=torch.bool)
                pad[:, :P] = self.prompt_mask == 0
                m = m | pad[:, None, None, :]
        self._rec["cross" if cross else "self"].append(eager_weights(qs, ks, m, self.dtype))
        return out

    def forward(self, inputs_embeds, enc_hidden, return_hidden=False):
        self._rec = dict(self=[], cross=[], hidden=[])
        B, q, _ = inputs_embeds.shape
        h0 = inputs_embeds
        if not self.cfg.rope_embeddings:
            h0 = inputs_embeds + self._p("embed_positions.weights").index_select(0, torch.arange(self.cur_len, self.cur_len + q))
        self._rec["hidden"].append(h0)
        # the outputs of layers 0 .. L-2: the residual stream entering layers 1 .. L-1, taken from the LayerNorm calls' inputs
        ln = self._ln
        seen = []

        def spy(x, name):
            if name.endswith("self_attn_layer_norm") and not name.startswith("layers.0."):
                seen.append(x)
            return ln(x, name)
        self._ln = spy
        try:
            logits, h = super().forward(inputs_embeds, enc_hidden, return_hidden=True)
        finally:
            self._ln = ln
        self._rec["hidden"] += seen + [h]
        self.calls.append(self._rec)
        return (logits, h) if return_hidden else logits

    def prefill(self, ids, enc_hidden, enc_mask, prompt_hidden, prompt_mask):
        self._enc_mask = enc_mask
        return super().prefill(ids, enc_hidden, enc_mask, prompt_hidden, prompt_mask)
