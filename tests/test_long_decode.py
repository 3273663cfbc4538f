"""The decode paths over full-length generations: caches up to position 4095 (max_position_embeddings - 1), where the product
runs them (generate() defaults to max_length 2580; the Large benchmark decodes to position 4095).

(a) Mini layer shape, B = 32: the cluster step kernel (step2.cu), the one-CTA-per-SM step kernel (step.cu, PTTS_STEP=legacy) and
    the multi-kernel path (PTTS_FUSED=0: attention_decode_kernel, sample.cu's one-row sampler) give the same tokens at every
    column and the same logits bits every 512 steps and at the last step, greedy and sampled (top-k 50).  The sampled run also
    pits the fused kernels' 3-rows-per-CTA sampler against sample.cu's 1-row pass at V = 1088.
(b) Large layer shape (H 1536, 24 heads), B = 32: the fused step kernel against the multi-kernel path, bit for bit.
(c) The multi-kernel path on narrow models against OracleDecoder, teacher-forced, after a left-padded prompt of 4000 positions
    up to position 4095 (sinusoidal table rows, rotary angles and GQA at long positions).
"""
import numpy as np
import pytest
import torch

from oracle.config import large_cfg, mini_cfg, tiny_cfg, tiny_dac_cfg
from oracle.decoder import OracleDecoder
from oracle.sampling import generate_tokens
from oracle.weights import make_dac_weights, make_decoder_weights
from tests.helpers import build_product_model, synth_inputs

pytestmark = pytest.mark.gpu

LAST_POS = 4095
CHECK_EVERY = 512


def _generate(cfg, w, B, S, P, mode, monkeypatch, do_sample):
    """Prompt of P positions, then decode until the step at position LAST_POS: raw ids [B*K, L] and the logits after every
    CHECK_EVERY-th step and after the last one."""
    monkeypatch.delenv("PTTS_STEP", raising=False)
    monkeypatch.delenv("PTTS_FUSED", raising=False)
    if mode == "legacy":
        monkeypatch.setenv("PTTS_STEP", "legacy")
    elif mode == "multi":
        monkeypatch.setenv("PTTS_FUSED", "0")
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16)
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=15)
    L = LAST_POS - P + 2          # the last decode step runs at position P + L - 2
    steps = L - 2
    sess = model.decoder.engine.session(B, P, S, P + L - 1)
    sess.begin(L, do_sample=do_sample, top_k=50 if do_sample else 0, seed=5, min_new_tokens=L, suppress_special=True,
               codebook_size=cfg.codebook_size)
    sess.prefill(prompt.to("cuda"), prompt_mask, enc.to("cuda"), enc_mask)
    fused = sess.fused
    sess.sample()
    logits, done = [], 0
    while done < steps:
        n = min(CHECK_EVERY, steps - done)
        sess.decode_steps(n)
        done += n
        logits.append(sess.logits.float().cpu().numpy().copy())
    torch.cuda.synchronize()
    raw =sess.raw_ids[:, :L].cpu().numpy().copy()
    sess.close()
    del model
    torch.cuda.empty_cache()
    return fused, raw, np.stack(logits)


def _assert_same(name, runs):
    base_mode, (_, raw0, lg0) = next(iter(runs.items()))
    for mode, (_, raw, lg) in runs.items():
        diff = np.nonzero((raw != raw0).any(0))[0]
        assert diff.size == 0, f"{name}: {mode} and {base_mode} tokens first differ at column {diff[:1]}"
        bad = [i for i in range(len(lg)) if not np.array_equal(lg[i].view(np.uint32), lg0[i].view(np.uint32))]
        assert not bad, f"{name}: {mode} and {base_mode} logits differ at checkpoints {bad} (every {CHECK_EVERY} steps)"


def _cluster_fits():
    return torch.cuda.get_device_properties(0).multi_processor_count >= 128


@pytest.mark.parametrize("shape", [{}, dict(hidden_size=768, num_attention_heads=12, ffn_dim=3072)], ids=["mini", "h768"])
@pytest.mark.parametrize("do_sample", [False, True], ids=["greedy", "topk50"])
def test_decode_paths_agree_to_position_4095(monkeypatch, shape, do_sample):
    cfg = mini_cfg(num_hidden_layers=2, max_position_embeddings=LAST_POS + 1, **shape)
    w = make_decoder_weights(cfg, seed=86, head_std=0.2)
    modes = ["legacy", "multi"] + (["cluster"] if _cluster_fits() else [])
    runs = {m: _generate(cfg, w, 32, 64, 32, m, monkeypatch, do_sample) for m in modes}
    kinds = {m: r[0] for m, r in runs.items()}
    assert kinds["legacy"] == 1 and kinds["multi"] == 0 and kinds.get("cluster", 2) == 2, kinds
    _assert_same(f"{'sampled' if do_sample else 'greedy'} {shape or 'mini'}", runs)


@pytest.mark.parametrize("do_sample", [False, True], ids=["greedy", "topk50"])
def test_large_step_kernel_equals_multi_kernel_to_position_4095(monkeypatch, do_sample):
    cfg = large_cfg(num_hidden_layers=2, max_position_embeddings=LAST_POS + 1)
    w = make_decoder_weights(cfg, seed=31, head_std=0.2)
    runs = {m: _generate(cfg, w, 32, 64, 32, m, monkeypatch, do_sample) for m in ("default", "multi")}
    assert runs["default"][0] in (1, 2) and runs["multi"][0] == 0, {m: r[0] for m, r in runs.items()}
    _assert_same(f"large {'sampled' if do_sample else 'greedy'}", runs)


def _long_variant(name):
    kw = dict(max_position_embeddings=LAST_POS + 1)
    if name == "abs":
        return tiny_cfg(**kw)
    if name == "rope":
        return tiny_cfg(rope_embeddings=True, **kw)
    if name == "gqa":
        return tiny_cfg(rope_embeddings=True, num_attention_heads=4, num_key_value_heads=2, num_cross_attention_key_value_heads=1,
                        hidden_size=256, **kw)
    return tiny_cfg(hidden_size=256, num_attention_heads=4, rope_embeddings=True, **kw)   # bf16 MHA: the tensor-core prefill sweep


P_LONG = 4000
STEPS_LONG = LAST_POS - P_LONG + 1   # teacher-forced steps: the last one runs at position P + STEPS - 1 = 4095


def _teacher_forced_long(cfg, dtype, seed):
    """OracleDecoder's greedy history (B = 2, S = 9, a left-padded prompt of P_LONG positions), replayed through the session as
    forced tokens; the session's cache holds exactly the positions 0 .. 4095 that max_position_embeddings allows."""
    B, S, P, L = 2, 9, P_LONG, STEPS_LONG + 1
    w = make_decoder_weights(cfg, seed=seed, head_std=0.3)
    model = build_product_model(cfg, tiny_dac_cfg(), w, make_dac_weights(tiny_dac_cfg(), seed=1), dtype=dtype)
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=seed)
    if dtype == torch.bfloat16:
        enc, prompt = enc.bfloat16().float(), prompt.bfloat16().float()
    ref = generate_tokens(OracleDecoder(cfg, w, dtype), cfg, enc, enc_mask, prompt, prompt_mask, dict(max_length=L, do_sample=False),
                          collect_logits=True)
    raw = ref["raw_ids"]
    sess = model.decoder.engine.session(B, P, S, P + L - 1)
    sess.begin(L, do_sample=False)
    sess.prefill(prompt.to("cuda"), prompt_mask, enc.to("cuda"), enc_mask)
    assert sess.fused == 0
    got = []
    for t in range(raw.shape[1] - 1):
        if t > 0:
            sess.decode_forward()
        got.append(sess.logits.float().cpu().numpy().copy())
        sess.sample(forced=torch.from_numpy(raw[:, t + 1].copy()))
    torch.cuda.synchronize()
    assert len(got) == STEPS_LONG
    return ref, got, sess.raw_ids[:, : raw.shape[1]].cpu().numpy()


@pytest.mark.parametrize("name", ["abs", "rope", "gqa"])
def test_multi_kernel_path_matches_oracle_at_long_positions_fp32(monkeypatch, name):
    monkeypatch.setenv("PTTS_FUSED", "0")
    ref, got, gpu_raw = _teacher_forced_long(_long_variant(name), torch.float32, seed=21)
    assert np.array_equal(gpu_raw, ref["raw_ids"])
    for t, (a, b) in enumerate(zip(got, ref["logits"])):
        err = np.abs(a - b).max()
        assert err < 2e-4, (name, t, err)
        assert np.array_equal(a.argmax(-1), b.argmax(-1)), (name, t)


def test_multi_kernel_path_matches_oracle_at_long_positions_bf16(monkeypatch):
    monkeypatch.setenv("PTTS_FUSED", "0")
    ref, got, gpu_raw = _teacher_forced_long(_long_variant("mha256"), torch.bfloat16, seed=22)
    assert np.array_equal(gpu_raw, ref["raw_ids"])
    for t, (a, b) in enumerate(zip(got, ref["logits"])):
        scale = np.abs(b).max()
        err = np.abs(a - b).max()
        assert err < 0.04 * scale, (t, err, scale)
        srt = np.sort(b, axis=-1)
        clear = (srt[:, -1] - srt[:, -2]) > 0.05 * scale
        assert np.array_equal(a.argmax(-1)[clear], b.argmax(-1)[clear]), t
