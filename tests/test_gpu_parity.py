"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI, against the CPU oracle.

Bars (stated per test): integer / index work bit-exact; fp32 model dtype within 2e-4 abs on logits and
exact greedy tokens; bf16 model dtype within bf16 resolution on logits and exact argmax wherever the
oracle's top-2 margin exceeds the tolerance; waveform RMS error < 1e-3 (BASELINE.json north_star).
"""
import os

import numpy as np
import pytest
import torch

from oracle.config import tiny_cfg, tiny_dac_cfg, mini_cfg, dac_cfg
from oracle.weights import make_decoder_weights, make_dac_weights
from oracle.decoder import OracleDecoder
from oracle.dac import OracleDAC
from oracle import delay_pattern as odp
from oracle.sampling import (ParlerLogitsProcessorOracle, generate_tokens, frames_from_raw, process_scores,
                             softmax_rows, valid_frame_mask)
from tests.helpers import build_product_model, synth_inputs, rms, product_decoder_config

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ---- integer operators: bit-exact ---------------------------------------------------------------
def test_delay_pattern_ops_bit_exact(golden_dir):
    from parler_tts_b200 import build_delay_pattern_mask, apply_delay_pattern_mask
    z = np.load(os.path.join(golden_dir, "delay_pattern.npz"))
    for ci in range(int(z["n"])):
        B, K, seq, L = (int(v) for v in z[f"c{ci}_meta"])
        ids = torch.from_numpy(z[f"c{ci}_ids"]).to(DEV)
        d, m = build_delay_pattern_mask(ids, 65, 64, L, K)
        assert np.array_equal(m.cpu().numpy(), z[f"c{ci}_mask"]), ci
        assert np.array_equal(d.cpu().numpy(), z[f"c{ci}_delayed"]), ci
        full = torch.from_numpy(z[f"c{ci}_full"]).to(DEV)
        assert np.array_equal(apply_delay_pattern_mask(full, m).cpu().numpy(), z[f"c{ci}_applied"])
        half = full[:, : max(1, L // 2)].contiguous()
        assert np.array_equal(apply_delay_pattern_mask(half, m).cpu().numpy(), z[f"c{ci}_applied_half"])


def test_logits_processor_op_bit_exact(golden_dir):
    from parler_tts_b200 import ParlerTTSLogitsProcessor
    z = np.load(os.path.join(golden_dir, "logits_processor.npz"))
    B, K, V, eos, steps = (int(v) for v in z["meta"])
    proc = ParlerTTSLogitsProcessor(eos, K, B, DEV)
    for s in range(steps):
        ids = torch.from_numpy(z["ids"][:, : s + 1].copy()).to(DEV)
        scores = torch.from_numpy(z["scores_in"][s].copy()).to(DEV)
        out = proc(ids, scores)
        assert out.data_ptr() == scores.data_ptr()  # in place, like the reference
        assert np.array_equal(out.cpu().numpy(), z["scores_out"][s]), s
        assert np.array_equal(proc.first_codebooks_unfinished.cpu().numpy(), z["first"][s]), s


def test_logits_processor_rejects_bad_eos():
    from parler_tts_b200 import ParlerTTSLogitsProcessor
    with pytest.raises(ValueError):
        ParlerTTSLogitsProcessor(-1, 4, 2, DEV)


# ---- decoder: teacher-forced logits and greedy tokens ------------------------------------------------
def _variant(name):
    if name == "abs":
        return tiny_cfg()
    if name == "rope":
        return tiny_cfg(rope_embeddings=True)
    return tiny_cfg(rope_embeddings=True, num_attention_heads=4, num_key_value_heads=2,
                    num_cross_attention_key_value_heads=1, hidden_size=256)


def _run_teacher_forced(cfg, dtype, B, S, P, steps, masks, seed, head_std=0.3):
    w = make_decoder_weights(cfg, seed=seed, head_std=head_std)
    dw = make_dac_weights(tiny_dac_cfg(), seed=1)
    model = build_product_model(cfg, tiny_dac_cfg(), w, dw, dtype=dtype)
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=seed, masks=masks)
    if dtype == torch.bfloat16:
        enc, prompt = enc.bfloat16().float(), (None if prompt is None else prompt.bfloat16().float())
    dec = OracleDecoder(cfg, w, dtype)
    L = steps + 1
    ref = generate_tokens(dec, cfg, enc, enc_mask, prompt, prompt_mask, dict(max_length=L, do_sample=False), collect_logits=True)
    raw = ref["raw_ids"]
    sess = model.decoder.engine.session(B, P, S, P + L)
    sess.begin(L, do_sample=False)
    sess.prefill(None if prompt is None else prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
    got_logits = []
    n = raw.shape[1] - 1
    for t in range(n):
        if t > 0:
            sess.decode_forward()
        got_logits.append(sess.logits.float().cpu().numpy().copy())
        sess.sample(forced=torch.from_numpy(raw[:, t + 1].copy()))
    torch.cuda.synchronize()
    gpu_raw = sess.raw_ids[:, : raw.shape[1]].cpu().numpy()
    return ref, got_logits, gpu_raw


@pytest.mark.parametrize("name", ["abs", "rope", "gqa"])
@pytest.mark.parametrize("masks", [True, False])
def test_decoder_teacher_forced_fp32(name, masks):
    cfg = _variant(name)
    ref, got, gpu_raw = _run_teacher_forced(cfg, torch.float32, B=3, S=9, P=5, steps=12, masks=masks, seed=11)
    assert np.array_equal(gpu_raw, ref["raw_ids"])  # forced history incl. finished-row padding, bit-exact
    for t, (a, b) in enumerate(zip(got, ref["logits"])):
        err = np.abs(a - b).max()
        assert err < 2e-4, (name, masks, t, err)
        assert np.array_equal(a.argmax(-1), b.argmax(-1)), (name, t)


@pytest.mark.parametrize("name", ["abs", "rope"])
def test_decoder_teacher_forced_bf16(name):
    cfg = _variant(name)
    ref, got, gpu_raw = _run_teacher_forced(cfg, torch.bfloat16, B=3, S=9, P=5, steps=12, masks=True, seed=12)
    assert np.array_equal(gpu_raw, ref["raw_ids"])
    for t, (a, b) in enumerate(zip(got, ref["logits"])):
        scale = np.abs(b).max()
        err = np.abs(a - b).max()
        assert err < 0.04 * scale, (name, t, err, scale)  # a few bf16 ulps of the largest logit
        srt = np.sort(b, axis=-1)
        clear = (srt[:, -1] - srt[:, -2]) > 0.05 * scale
        assert np.array_equal(a.argmax(-1)[clear], b.argmax(-1)[clear]), (name, t)


def test_no_prompt_prefix():
    cfg = tiny_cfg()
    ref, got, gpu_raw = _run_teacher_forced(cfg, torch.float32, B=2, S=6, P=0, steps=8, masks=False, seed=13)
    for a, b in zip(got, ref["logits"]):
        assert np.abs(a - b).max() < 2e-4


def test_greedy_free_running_tokens_exact():
    """Device-resident loop (CUDA graph replay, no host sync) == oracle loop, token for token (fp32)."""
    cfg = tiny_cfg()
    w = make_decoder_weights(cfg, seed=22, head_std=0.5)  # seed chosen so the oracle's smallest top-2 margin is 6.9e-3
    model = build_product_model(cfg, tiny_dac_cfg(), w, make_dac_weights(tiny_dac_cfg(), seed=1), dtype=torch.float32)
    B, S, P, L = 4, 8, 4, 40
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=3)
    dec = OracleDecoder(cfg, w, torch.float32)
    ref = generate_tokens(dec, cfg, enc, enc_mask, prompt, prompt_mask, dict(max_length=L, do_sample=False), collect_logits=True)
    sess = model.decoder.engine.session(B, P, S, P + L)
    sess.begin(L, do_sample=False)
    sess.prefill(prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
    sess.sample()
    sess.decode_steps(L - 2)
    torch.cuda.synchronize()
    n = ref["raw_ids"].shape[1]
    st = sess.state.cpu().numpy()
    got = sess.raw_ids[:, :n].cpu().numpy()
    margins = [np.sort(s, -1)[:, -1] - np.sort(s, -1)[:, -2] for s in ref["scores"]]
    assert min(m.min() for m in margins) > 1e-3, "test weights give near-ties; pick another seed"
    assert np.array_equal(got, ref["raw_ids"])
    assert int(st[0]) == n  # stopped at the same length (EOS / max_length), decided on the device


def test_eos_and_ragged_finish():
    """Rows finish independently; finished rows emit pad; processor gates EOS by codebook (Q11, Q12)."""
    cfg = tiny_cfg()
    w = make_decoder_weights(cfg, seed=31, head_std=0.5)
    for k in range(cfg.num_codebooks):  # make EOS likely
        w[f"decoder.lm_heads.{k}.weight"][cfg.eos_token_id] *= 6.0
    model = build_product_model(cfg, tiny_dac_cfg(), w, make_dac_weights(tiny_dac_cfg(), seed=1), dtype=torch.float32)
    B, S, P, L = 4, 8, 4, 48
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=4)
    dec = OracleDecoder(cfg, w, torch.float32)
    ref = generate_tokens(dec, cfg, enc, enc_mask, prompt, prompt_mask, dict(max_length=L, do_sample=False))
    assert (ref["raw_ids"] == cfg.eos_token_id).any(), "fixture should exercise EOS"
    sess = model.decoder.engine.session(B, P, S, P + L)
    sess.begin(L, do_sample=False)
    sess.prefill(prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
    sess.sample()
    sess.decode_steps(L - 2)
    torch.cuda.synchronize()
    n = ref["raw_ids"].shape[1]
    assert int(sess.state[0].item()) == n
    assert np.array_equal(sess.raw_ids[:, :n].cpu().numpy(), ref["raw_ids"])


# ---- sampling -------------------------------------------------------------------------------------
@pytest.mark.parametrize("gen", [dict(do_sample=True, top_k=10), dict(do_sample=True, top_k=0, top_p=0.8, temperature=0.7),
                                 dict(do_sample=True, top_k=20, top_p=0.9, temperature=1.3, min_new_tokens=5)])
def test_processed_scores_match_oracle(gen):
    """Warper chain on the device == oracle chain: same kept set, same values (fp32 exact except cumsum edge)."""
    cfg = tiny_cfg()
    w = make_decoder_weights(cfg, seed=41, head_std=0.6)
    model = build_product_model(cfg, tiny_dac_cfg(), w, make_dac_weights(tiny_dac_cfg(), seed=1), dtype=torch.float32)
    B, S, P, L = 3, 8, 4, 12
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=5)
    sess = model.decoder.engine.session(B, P, S, P + L)
    sess.begin(L, seed=7, **gen)
    sess.prefill(prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
    parler = ParlerLogitsProcessorOracle(cfg.eos_token_id, cfg.num_codebooks, B)
    for t in range(L - 1):
        if t > 0:
            sess.decode_forward()
        logits = sess.logits.cpu().numpy().copy()
        raw = sess.raw_ids[:, : t + 1].cpu().numpy()
        sess.sample()
        torch.cuda.synchronize()
        got = sess.scores.cpu().numpy()
        want = process_scores(logits, raw, parler, dict(gen))
        kept_g, kept_w = np.isfinite(got), np.isfinite(want)
        diff = kept_g != kept_w
        assert diff.sum() <= 1, (t, diff.sum())  # at most one borderline top-p token per call
        both = kept_g & kept_w
        assert np.abs(got[both] - want[both]).max() < 1e-5
        tok = sess.raw_ids[:, t + 1].cpu().numpy()
        fin = raw.shape[1] > 0
        for r in range(tok.shape[0]):
            assert kept_g[r, tok[r]] or tok[r] == cfg.pad_token_id


def test_sampling_distribution():
    """Philox inverse-CDF draws follow the processed distribution (chi-square over many seeds)."""
    cfg = tiny_cfg()
    w = make_decoder_weights(cfg, seed=43, head_std=0.6)
    model = build_product_model(cfg, tiny_dac_cfg(), w, make_dac_weights(tiny_dac_cfg(), seed=1), dtype=torch.float32)
    B, S, P, L = 2, 6, 3, 4
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=6, masks=False)
    sess = model.decoder.engine.session(B, P, S, P + L)
    counts = None
    N = 400
    for seed in range(N):
        sess.begin(L, do_sample=True, top_k=8, seed=seed)
        sess.prefill(prompt.to(DEV), None, enc.to(DEV), None)
        sess.sample()
        tok = sess.raw_ids[:, 1].cpu().numpy()
        if counts is None:
            probs = softmax_rows(sess.scores.cpu().numpy())
            counts = np.zeros_like(probs)
        counts[np.arange(tok.shape[0]), tok] += 1
    for r in range(counts.shape[0]):
        nz = probs[r] > 0
        assert counts[r][~nz].sum() == 0
        exp = probs[r][nz] * N
        chi2 = ((counts[r][nz] - exp) ** 2 / np.maximum(exp, 1e-9)).sum()
        assert chi2 < 40.0, (r, chi2)  # 7 dof; p ~ 1e-6
    # same seed -> same draw; shard-invariance: a row's stream depends only on (seed, row, column)
    sess.begin(L, do_sample=True, top_k=8, seed=5)
    sess.prefill(prompt.to(DEV), None, enc.to(DEV), None)
    sess.sample()
    a = sess.raw_ids[:, 1].cpu().numpy().copy()
    sess.begin(L, do_sample=True, top_k=8, seed=5)
    sess.prefill(prompt.to(DEV), None, enc.to(DEV), None)
    sess.sample()
    assert np.array_equal(a, sess.raw_ids[:, 1].cpu().numpy())


# ---- DAC ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_dac_decode_tiny(golden_dir, dtype):
    from parler_tts_b200 import DACModel
    from tests.helpers import product_dac_config
    z = np.load(os.path.join(golden_dir, "dac_decode.npz"))
    dcfg = tiny_dac_cfg()
    m = DACModel(product_dac_config(dcfg), DEV, dtype).load_state_dict(make_dac_weights(dcfg, seed=2))
    codes = torch.from_numpy(z["codes"]).to(DEV)
    audio = m.decode(codes[None], [None, None]).audio_values
    assert audio.shape == (2, 1, 11 * 512)
    ref = z["audio"].reshape(2, 1, -1)  # produced by transformers' DacModel in the build container
    err = rms(audio.float().cpu().numpy() - ref)
    if dtype == torch.float32:
        assert err < 1e-5, err
    else:
        # bf16 storage (quirk Q16): as accurate as torch's own bf16 run of the same network on the CPU
        cpu_bf16 = OracleDAC(dcfg, make_dac_weights(dcfg, seed=2), torch.bfloat16).decode(torch.from_numpy(z["codes"])[None]).float().numpy()
        err_cpu = rms(cpu_bf16 - ref)
        assert err < 1.5 * err_cpu + 1e-3, (err, err_cpu)
        assert err < 0.1 * rms(ref), (err, rms(ref))
    with pytest.raises(ValueError):
        m.decode(torch.cat([codes[None], codes[None]]), [None])  # "Expected one frame"
    with pytest.raises(IndexError):
        m.decode((codes + dcfg.codebook_size)[None], [None])


def test_dac_decode_real_shape_fp32():
    """44.1 kHz DAC shape (1536 -> 96 channels, hop 512), short clip; waveform RMS error < 1e-3 (north_star bar)."""
    from parler_tts_b200 import DACModel
    from tests.helpers import product_dac_config
    dcfg = dac_cfg()
    w = make_dac_weights(dcfg, seed=3)
    m = DACModel(product_dac_config(dcfg), DEV, torch.float32).load_state_dict(w)
    g = torch.Generator().manual_seed(9)
    codes = torch.randint(0, 1024, (2, 9, 7), generator=g)
    ref = OracleDAC(dcfg, w).decode(codes[None]).numpy()
    got = m.decode(codes[None].to(DEV), [None]).audio_values.cpu().numpy()
    assert got.shape == ref.shape == (2, 1, 7 * 512)
    assert rms(ref) > 1e-3
    assert rms(got - ref) < 1e-4, rms(got - ref)


# ---- end to end ----------------------------------------------------------------------------------
def test_generate_end_to_end_fp32():
    """generate(): tokens bit-exact vs the oracle loop, waveform within 1e-3 RMS, ragged lengths equal."""
    cfg, dcfg = tiny_cfg(), tiny_dac_cfg()
    w = make_decoder_weights(cfg, seed=51, head_std=0.5)
    for k in range(cfg.num_codebooks):
        w[f"decoder.lm_heads.{k}.weight"][cfg.eos_token_id] *= 3.0
    dw = make_dac_weights(dcfg, seed=2)
    model = build_product_model(cfg, dcfg, w, dw, dtype=torch.float32)
    B, S, P, L = 3, 8, 4, 30
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=8)
    audio, out = model.generate(encoder_outputs=(enc.to(DEV),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV),
                                prompt_attention_mask=prompt_mask.to(DEV), do_sample=False, max_length=L, return_codes=True)
    dec = OracleDecoder(cfg, w, torch.float32)
    ref = generate_tokens(dec, cfg, enc, enc_mask, prompt, prompt_mask, dict(max_length=L, do_sample=False))
    codes = frames_from_raw(ref["raw_ids"], ref["delay_mask"], cfg, B)
    assert np.array_equal(out.audio_codes.cpu().numpy(), codes)
    dac = OracleDAC(dcfg, dw)
    for b in range(B):
        ok = valid_frame_mask(codes[b:b + 1], dcfg.codebook_size)[0]
        if ok.sum() == 0:
            assert out.audios_length[b] == 1
            continue
        refa = dac.decode(torch.from_numpy(codes[b:b + 1][:, :, ok])[None]).numpy().reshape(-1)
        assert out.audios_length[b] == refa.shape[0]
        got = audio[b, : refa.shape[0]].float().cpu().numpy()
        assert rms(got - refa) < 1e-3
        assert float(audio[b, refa.shape[0]:].abs().sum()) == 0.0  # zero padding to the longest (:3643-3647)


def test_streamer_batch1():
    from parler_tts_b200 import ParlerTTSStreamer
    cfg, dcfg = tiny_cfg(), tiny_dac_cfg()
    w = make_decoder_weights(cfg, seed=61, head_std=0.5)
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=torch.float32)
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, 1, 6, 3, seed=9, masks=False)
    st = ParlerTTSStreamer(model, device=DEV, play_steps=8)
    audio = model.generate(encoder_outputs=(enc.to(DEV),), prompt_hidden_states=prompt.to(DEV), do_sample=False, max_length=26,
                           streamer=st, _suppress_special=True)
    chunks = [c for c in st]
    total = np.concatenate(chunks)
    full = audio[0].float().cpu().numpy()
    assert len(chunks) >= 2 and total.shape[0] == full.shape[0]
    with pytest.raises(ValueError):
        st.put(torch.zeros(2 * cfg.num_codebooks, dtype=torch.long))


# ---- Mini shape (BASELINE configs[0] / configs[1] shapes at reduced step counts) ----------------------
def test_mini_shape_fp32_greedy_b1():
    """BASELINE configs[0]: Mini fp32 greedy B=1 -- tokens match the CPU oracle exactly over 24 steps."""
    cfg = mini_cfg(max_position_embeddings=256)
    w = make_decoder_weights(cfg, seed=71, head_std=0.2)
    model = build_product_model(cfg, tiny_dac_cfg(n_codebooks=9, codebook_size=1024), w,
                                make_dac_weights(tiny_dac_cfg(n_codebooks=9, codebook_size=1024), seed=1), dtype=torch.float32)
    B, S, P, L = 1, 16, 8, 25
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=10, masks=False)
    dec = OracleDecoder(cfg, w, torch.float32)
    ref = generate_tokens(dec, cfg, enc, None, prompt, None, dict(max_length=L, do_sample=False), collect_logits=True)
    sess = model.decoder.engine.session(B, P, S, P + L)
    sess.begin(L, do_sample=False)
    sess.prefill(prompt.to(DEV), None, enc.to(DEV), None)
    l0 = sess.logits.cpu().numpy()
    assert np.abs(l0 - ref["logits"][0]).max() < 5e-4
    sess.sample()
    sess.decode_steps(L - 2)
    torch.cuda.synchronize()
    n = ref["raw_ids"].shape[1]
    assert np.array_equal(sess.raw_ids[:, :n].cpu().numpy(), ref["raw_ids"])


def test_mini_shape_bf16_batch32_teacher_forced():
    """BASELINE configs[1] shape (B=32, bf16), 6 teacher-forced steps vs the bf16 CPU oracle."""
    cfg = mini_cfg(max_position_embeddings=256)
    w = make_decoder_weights(cfg, seed=72, head_std=0.2)
    dcfg = tiny_dac_cfg(n_codebooks=9, codebook_size=1024)
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16)
    B, S, P, steps = 32, 16, 8, 6
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=11, masks=True)
    enc, prompt = enc.bfloat16().float(), prompt.bfloat16().float()
    dec = OracleDecoder(cfg, w, torch.bfloat16)
    L = steps + 1
    ref = generate_tokens(dec, cfg, enc, enc_mask, prompt, prompt_mask, dict(max_length=L, do_sample=False), collect_logits=True)
    sess = model.decoder.engine.session(B, P, S, P + L)
    sess.begin(L, do_sample=False)
    sess.prefill(prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
    agree = total = 0
    for t in range(steps):
        if t > 0:
            sess.decode_forward()
        a = sess.logits.float().cpu().numpy()
        b = ref["logits"][t]
        scale = np.abs(b).max()
        assert np.abs(a - b).max() < 0.05 * scale, (t, np.abs(a - b).max(), scale)
        srt = np.sort(b, -1)
        clear = (srt[:, -1] - srt[:, -2]) > 0.05 * scale
        assert np.array_equal(a.argmax(-1)[clear], b.argmax(-1)[clear])
        agree += int((a.argmax(-1) == b.argmax(-1)).sum())
        total += a.shape[0]
        sess.sample(forced=torch.from_numpy(ref["raw_ids"][:, t + 1].copy()))
    assert agree / total > 0.9


# ---- fused persistent step kernel (step.cu) vs the multi-kernel path -------------------------------
def _free_run_bf16(cfg, w, B, S, P, L, fused, monkeypatch, gen=None, seed=3):
    monkeypatch.setenv("PTTS_FUSED", "1" if fused else "0")
    monkeypatch.setenv("PTTS_STEP", "legacy")   # step.cu: the kernel that shares its reduction order with the multi-kernel path
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16)
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=seed)
    sess = model.decoder.engine.session(B, P, S, P + L)
    sess.begin(L, **(gen or dict(do_sample=False)))
    sess.prefill(prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
    sess.sample()
    sess.decode_steps(L - 2)
    torch.cuda.synchronize()
    n = int(sess.state[0].item())
    return sess.raw_ids[:, :n].cpu().numpy().copy(), sess.logits.cpu().numpy().copy(), sess.launches


@pytest.mark.parametrize("name", ["abs", "rope", "gqa"])
def test_fused_step_equals_multikernel_bitwise(name, monkeypatch):
    """Same arithmetic, same reduction order: tokens AND last-step logits are bit-identical."""
    cfg = _variant(name)
    w = make_decoder_weights(cfg, seed=81, head_std=0.5)
    a_ids, a_log, a_launch = _free_run_bf16(cfg, w, 5, 9, 5, 36, True, monkeypatch)
    b_ids, b_log, b_launch = _free_run_bf16(cfg, w, 5, 9, 5, 36, False, monkeypatch)
    assert a_ids.shape == b_ids.shape and np.array_equal(a_ids, b_ids)
    assert np.array_equal(a_log, b_log)
    assert a_launch < b_launch / 10  # one kernel per token instead of 8L+3


def test_fused_step_sampling_and_eos(monkeypatch):
    cfg = tiny_cfg()
    w = make_decoder_weights(cfg, seed=82, head_std=0.5)
    for k in range(cfg.num_codebooks):
        w[f"decoder.lm_heads.{k}.weight"][cfg.eos_token_id] *= 5.0
    gen = dict(do_sample=True, top_k=12, temperature=0.9, top_p=0.95, seed=11)
    a_ids, a_log, _ = _free_run_bf16(cfg, w, 4, 8, 4, 40, True, monkeypatch, gen)
    b_ids, b_log, _ = _free_run_bf16(cfg, w, 4, 8, 4, 40, False, monkeypatch, gen)
    assert (a_ids == cfg.eos_token_id).any()
    assert np.array_equal(a_ids, b_ids) and np.array_equal(a_log, b_log)


def test_fused_step_mini_shape_batch32(monkeypatch):
    """BASELINE configs[1] shape: fused kernel == multi-kernel path over 20 free-running greedy steps."""
    cfg = mini_cfg(max_position_embeddings=256)
    w = make_decoder_weights(cfg, seed=83, head_std=0.2)
    a_ids, a_log, _ = _free_run_bf16(cfg, w, 32, 16, 8, 22, True, monkeypatch)
    b_ids, b_log, _ = _free_run_bf16(cfg, w, 32, 16, 8, 22, False, monkeypatch)
    assert np.array_equal(a_ids, b_ids)
    assert np.array_equal(a_log, b_log)


# Mini (16 heads: 64 clusters of 2 CTAs) and a 12-head shape (H 768, F 3072: 48 clusters).  At H = 768 each K half of a rank's
# slice is an ODD number of k-tiles (3) and a K slice holds three heads, not four: the cases mma_slice's paired k-tile loop and the
# attention output placement must handle.  A 132-SM H100 holds 66 clusters of 2 co-resident: both shapes.
CLUSTER_SHAPES = {"mini": {}, "h768": dict(hidden_size=768, num_attention_heads=12, ffn_dim=3072)}
_cluster_fit = {}


def _cluster_shapes(monkeypatch):
    """The CLUSTER_SHAPES whose cluster grid this device holds co-resident (probed with a one-layer session: the grid depends on the
    head count only).  Shapes it cannot hold decode with step.cu and are reported, not run; at least one must fit."""
    monkeypatch.setenv("PTTS_STEP", "cluster")
    for name, kw in CLUSTER_SHAPES.items():
        if name not in _cluster_fit:
            cfg = mini_cfg(num_hidden_layers=1, max_position_embeddings=32, **kw)
            dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
            model = build_product_model(cfg, dcfg, make_decoder_weights(cfg, seed=1), make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16)
            enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, 32, 4, 2, seed=1)
            sess = model.decoder.engine.session(32, 2, 4, 8)
            sess.begin(4, do_sample=False)
            sess.prefill(prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
            _cluster_fit[name] = sess.fused == 2
    fits = [n for n in CLUSTER_SHAPES if _cluster_fit[n]]
    print(f"\n[cluster] shapes whose grid this device holds: {fits}; not co-resident (step.cu): "
          f"{[n for n in CLUSTER_SHAPES if not _cluster_fit[n]]}")
    assert fits, "the device holds none of the cluster grids"
    return fits


def test_cluster_step_kernel_matches_legacy_step_kernel(monkeypatch):
    """step2.cu (2 clusters x 4 CTAs per head, K split 8 ways, DSMEM exchange, attention fused into the projection phases) against
    step.cu, B=32, at every CLUSTER_SHAPES entry the device holds: same inputs, teacher-forced on the legacy kernel's greedy tokens.
    The two kernels add the same products in a different order, so the logits agree to bf16 accumulation noise and the greedy
    choice wherever it is clear."""
    for shape in _cluster_shapes(monkeypatch):
        _check_cluster_vs_legacy(monkeypatch, mini_cfg(num_hidden_layers=4, max_position_embeddings=256, **CLUSTER_SHAPES[shape]))


def _check_cluster_vs_legacy(monkeypatch, cfg):
    w = make_decoder_weights(cfg, seed=86, head_std=0.2)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    B, S, P, steps = 32, 24, 12, 40     # cache length 13 -> 53: several 16-key ring chunks per attention warp
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=15)
    L = steps + 2
    out = {}
    forced = None
    for mode in ("legacy", "cluster"):
        monkeypatch.setenv("PTTS_STEP", mode)
        model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16)
        sess = model.decoder.engine.session(B, P, S, P + L)
        sess.begin(L, do_sample=False)
        sess.prefill(prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
        assert sess.fused == (1 if mode == "legacy" else 2), (mode, sess.fused)
        logits, toks = [], []
        for t in range(steps):
            if t > 0:
                sess.decode_forward()
                logits.append(sess.logits.float().cpu().numpy().copy())
            sess.sample(forced=None if forced is None else torch.from_numpy(forced[:, t].copy()))
            toks.append(sess.raw_ids[:, t + 1].cpu().numpy().copy())
        torch.cuda.synchronize()
        out[mode] = (np.stack(logits), np.stack(toks, 1))
        if forced is None:
            forced = out[mode][1]
    a, b = out["cluster"][0], out["legacy"][0]
    scale = np.abs(b).max()
    assert np.isfinite(a).all()
    err = np.abs(a - b).max(axis=(1, 2)) / scale
    assert err.max() < 0.02, err
    srt = np.sort(b, -1)
    clear = (srt[..., -1] - srt[..., -2]) > 0.04 * scale
    assert np.array_equal(a.argmax(-1)[clear], b.argmax(-1)[clear])
    # free-running with the in-kernel sampler: runs to the end and stays finite
    monkeypatch.setenv("PTTS_STEP", "cluster")
    ids, lg, launches = _free_run_cluster(cfg, w, B, S, P, L, dict(do_sample=True, top_k=50, seed=5, min_new_tokens=L - 1, suppress_special=True, codebook_size=1024))
    assert ids.shape[1] == L and np.isfinite(lg).all() and (ids[:, 1:] < 1024).all()


def test_cluster_kernel_many_steps_per_launch_equals_one_step_per_launch(monkeypatch):
    """ptts_decode_steps(n) on the cluster kernel is ONE launch that loops over the tokens (cur_len, the unfinished count and the
    stop decision advance on the device).  Same tokens, same final logits, same stopping column as one launch per token --
    sampling included, and with an early finish inside a launch (EOS allowed after 6 tokens); at every CLUSTER_SHAPES entry the
    device holds."""
    for shape in _cluster_shapes(monkeypatch):
        monkeypatch.delenv("PTTS_STEP", raising=False)
        _check_many_steps_per_launch(monkeypatch, mini_cfg(num_hidden_layers=2, max_position_embeddings=96, **CLUSTER_SHAPES[shape]))


def _check_many_steps_per_launch(monkeypatch, cfg):
    w = make_decoder_weights(cfg, seed=9, head_std=0.6)
    B, S, P, L = 32, 12, 5, 40
    runs = {}
    for name, per_launch, gen in [("free", None, dict(do_sample=True, top_k=50, seed=5, min_new_tokens=L - 1, suppress_special=True, codebook_size=1024)),
                                  ("eos", None, dict(do_sample=True, top_k=0, temperature=1.5, seed=11, min_new_tokens=6))]:
        for per in ("1", "7", None):
            if per is None:
                monkeypatch.delenv("PTTS_STEPS_PER_LAUNCH", raising=False)
            else:
                monkeypatch.setenv("PTTS_STEPS_PER_LAUNCH", per)
            runs[(name, per)] = _free_run_cluster(cfg, w, B, S, P, L, gen, extra_steps=9)
        one = runs[(name, "1")]
        for per in ("7", None):
            got = runs[(name, per)]
            assert got[0].shape == one[0].shape, f"{name}: stopping column differs ({got[0].shape} vs {one[0].shape})"
            assert np.array_equal(got[0], one[0]), f"{name}: tokens differ with {per or 64} steps per launch"
            assert np.array_equal(got[1], one[1]), f"{name}: last logits differ"
        assert runs[(name, None)][2] < one[2]   # fewer launches
    assert runs[("free", "1")][0].shape[1] == L


def _free_run_cluster(cfg, w, B, S, P, L, gen, extra_steps=0):
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16)
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=3)
    sess = model.decoder.engine.session(B, P, S, P + L)
    sess.begin(L, **gen)
    sess.prefill(prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
    assert sess.fused == 2
    sess.sample()
    sess.decode_steps(L - 2 + extra_steps)   # (steps past the end must be no-ops: every row is finished at max_length)
    torch.cuda.synchronize()
    n = int(sess.state[0].item())
    return sess.raw_ids[:, :n].cpu().numpy().copy(), sess.logits.cpu().numpy().copy(), sess.launches


def test_dac_decode_real_shape_bf16_tensor_core(monkeypatch):
    """DAC decode in bf16: the wgmma implicit-GEMM path vs the fp32 oracle (and vs the SIMT bf16 path), at the 44.1 kHz shape
    (channel tiles of 128 and 96) and at decoder width 1280 with three blocks (1280 -> 640 -> 320 -> 160 channels), whose 320- and
    160-channel layers take the 64- and 32-column tiles of the wgmma pipeline."""
    from parler_tts_b200 import DACModel
    from tests.helpers import product_dac_config
    for dcfg in (dac_cfg(), dac_cfg(decoder_hidden_size=1280, upsampling_ratios=[8, 8, 4])):
        w = make_dac_weights(dcfg, seed=3)
        g = torch.Generator().manual_seed(9)
        codes = torch.randint(0, 1024, (2, 9, 5), generator=g)
        ref = OracleDAC(dcfg, w).decode(codes[None]).numpy()
        outs = {}
        for tc in ("1", "0"):
            monkeypatch.setenv("PTTS_DAC_TC", tc)
            m = DACModel(product_dac_config(dcfg), DEV, torch.bfloat16).load_state_dict(w)
            outs[tc] = m.decode(codes[None].to(DEV), [None]).audio_values.float().cpu().numpy()
            assert outs[tc].shape == ref.shape
        e_tc, e_simt = rms(outs["1"] - ref), rms(outs["0"] - ref)
        # bf16 storage between layers dominates both; the tensor-core path must be no worse than the FMA path
        assert e_tc < 0.1 * rms(ref) + 1e-3, (dcfg.decoder_hidden_size, e_tc, rms(ref))
        assert e_tc < 1.5 * e_simt + 1e-3, (dcfg.decoder_hidden_size, e_tc, e_simt)


def test_streamer_incremental_equals_full_decode():
    """ParlerTTSStreamer(incremental=True) (SURVEY 8f rank 1): chunks decoded from `new frames + receptive-field context` windows
    concatenate to the waveform generate() returns from one decode of all frames.  (Host logic verified on the CPU against the
    oracle DAC in tests/test_host_logic.py; added after the last GPU session of round 1: first exercised by the round-end run.)"""
    from parler_tts_b200 import ParlerTTSStreamer
    cfg, dcfg = tiny_cfg(), tiny_dac_cfg()
    w = make_decoder_weights(cfg, seed=61, head_std=0.5)
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=torch.float32)
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, 1, 6, 3, seed=9, masks=False)
    st = ParlerTTSStreamer(model, device=DEV, play_steps=6, incremental=True)
    audio = model.generate(encoder_outputs=(enc.to(DEV),), prompt_hidden_states=prompt.to(DEV), do_sample=False, max_length=60,
                           streamer=st, _suppress_special=True)
    chunks = [c for c in st]
    total = np.concatenate(chunks)
    full = audio[0].float().cpu().numpy()
    assert total.shape[0] == full.shape[0] and sum(len(c) > 0 for c in chunks) >= 2
    assert np.abs(total - full).max() < 1e-4


def test_fused_step_large_shape_single_tile_buffer(monkeypatch):
    """Parler-TTS-Large layer shape (H=1536, F=6144, 24 heads; 2 layers): the fused kernel runs with ONE activation tile buffer,
    a 96 KB weight slice per task and matrices whose tasks wrap around the grid (fc2: 192 tasks on one CTA per SM) -- the code
    paths the Mini shape does not reach.  Same bar as the other shapes: bit-identical to the multi-kernel path.
    (Added after the last GPU session of round 1: first exercised by the round-end run.)"""
    from oracle.config import large_cfg
    cfg = large_cfg(num_hidden_layers=2, max_position_embeddings=128)
    w = make_decoder_weights(cfg, seed=84, head_std=0.2)
    a_ids, a_log, a_launch = _free_run_bf16(cfg, w, 8, 12, 6, 14, True, monkeypatch)
    b_ids, b_log, b_launch = _free_run_bf16(cfg, w, 8, 12, 6, 14, False, monkeypatch)
    assert a_launch < b_launch / 3, (a_launch, b_launch)  # the fused kernel was really used
    assert np.array_equal(a_ids, b_ids)
    assert np.array_equal(a_log, b_log)
