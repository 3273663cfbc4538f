"""CPU restatement of config.prompt_cross_attention (test infrastructure only).

  prompt states       embed_prompts(prompt_input_ids) + embed_positions[0:P] in the model dtype (:3102-3104, :2792-2794)
  masks               one given: the other becomes ones; neither: no mask (:3110-3117)
  concatenation       [description states || prompt states] and [description mask || prompt mask] along the keys (:3120-3122)
  decoder             no prompt prefix: OracleDecoder.prefill(..., prompt_hidden=None) over the S + P keys
Built on the oracle's own pieces (oracle/weights.py sinusoidal_table); tests/golden/prompt_cross.npz pins it against the
reference's code.
"""
from __future__ import annotations
import torch
import torch.nn.functional as F

from oracle.weights import sinusoidal_table


def assemble(enc_hidden, enc_mask, prompt_ids, prompt_mask, embed_prompts, max_position_embeddings: int, dtype=torch.float32):
    """-> (encoder states [B, S + P, H] in dtype, mask [B, S + P] or None)."""
    B, S, H = enc_hidden.shape
    P = prompt_ids.shape[1]
    positions = sinusoidal_table(max_position_embeddings, H).to(dtype)
    prompt = F.embedding(prompt_ids, embed_prompts.to(dtype)) + positions[:P]
    if prompt_mask is not None and enc_mask is None:
        enc_mask = torch.ones(B, S, dtype=prompt_mask.dtype)
    elif enc_mask is not None and prompt_mask is None:
        prompt_mask = torch.ones(B, P, dtype=enc_mask.dtype)
    states = torch.cat([enc_hidden.to(dtype), prompt], dim=1)
    return states, (None if prompt_mask is None else torch.cat([enc_mask, prompt_mask], dim=1))
