"""The benchmarked decoder (Parler-TTS-Mini, bf16, batch 32) decodes with the cluster step kernel (step2.cu) by default: its grid of
64 clusters of 2 CTAs is co-resident on a 132-SM H100 (one cluster per TPC, 66 in all).  The cluster kernel reproduces the
one-CTA-per-SM step kernel (step.cu) bit for bit, so which of the two a device runs does not change any output."""
import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_dac_cfg
from oracle.weights import make_decoder_weights, make_dac_weights
from tests.helpers import build_product_model, synth_inputs

pytestmark = pytest.mark.gpu


def _need_132_sm_class_device():
    props = torch.cuda.get_device_properties(0)
    if props.multi_processor_count < 128:
        pytest.skip(f"{props.name} has {props.multi_processor_count} SMs: fewer than the 64 co-resident clusters of 2 Mini needs")


def test_mini_batch32_session_runs_the_cluster_step_kernel(monkeypatch):
    _need_132_sm_class_device()
    monkeypatch.delenv("PTTS_STEP", raising=False)
    cfg = mini_cfg(num_hidden_layers=1, max_position_embeddings=32)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    model = build_product_model(cfg, dcfg, make_decoder_weights(cfg, seed=1), make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16)
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, 32, 4, 2, seed=1)
    sess = model.decoder.engine.session(32, 2, 4, 8)
    sess.begin(4, do_sample=False)
    sess.prefill(prompt.to("cuda"), prompt_mask, enc.to("cuda"), enc_mask)
    assert sess.fused == 2, f"fused kind {sess.fused}: Mini at batch 32 does not decode with the cluster step kernel"


@pytest.mark.parametrize("shape", [{}, dict(hidden_size=768, num_attention_heads=12, ffn_dim=3072)], ids=["mini", "h768"])
def test_cluster_step_kernel_equals_legacy_step_kernel_bitwise(monkeypatch, shape):
    """Greedy logits of every step and the tokens of an in-kernel top-k run (many steps per launch), B = 32, a cache long enough
    for several 32-key attention chunks per warp: identical bits from step2.cu and step.cu."""
    _need_132_sm_class_device()
    cfg = mini_cfg(num_hidden_layers=2, max_position_embeddings=128, **shape)
    w = make_decoder_weights(cfg, seed=86, head_std=0.2)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    B, S, P, steps = 32, 40, 12, 60
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=15)
    L = steps + 2
    out = {}
    for mode in ("legacy", "cluster"):
        monkeypatch.setenv("PTTS_STEP", mode)
        model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16)
        sess = model.decoder.engine.session(B, P, S, P + L)
        sess.begin(L, do_sample=False)
        sess.prefill(prompt.to("cuda"), prompt_mask, enc.to("cuda"), enc_mask)
        assert sess.fused == (1 if mode == "legacy" else 2), (mode, sess.fused)
        logits = []
        sess.sample()
        for _ in range(1, steps):
            sess.decode_forward()
            logits.append(sess.logits.float().cpu().numpy().copy())
            sess.sample()
        greedy = sess.raw_ids[:, : steps + 1].cpu().numpy().copy()
        sess.begin(L, do_sample=True, top_k=50, seed=5, min_new_tokens=steps, suppress_special=True, codebook_size=1024)
        sess.prefill(prompt.to("cuda"), prompt_mask, enc.to("cuda"), enc_mask)
        sess.sample()
        sess.decode_steps(steps - 1)
        torch.cuda.synchronize()
        out[mode] = (np.stack(logits), greedy, sess.raw_ids[:, : steps + 1].cpu().numpy().copy())
    for name, a, b in zip(("logits", "greedy tokens", "sampled tokens"), out["cluster"], out["legacy"]):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), f"{name} differ between the two step kernels"
