"""generate(return_dict_in_generate=True, output_scores=True, output_logits=True): the per-step rows the sampler records.

Host tests: the GenerationConfig fields, the keyword handling and the chunk / window arithmetic.  GPU tests: the recorded rows
bit-identical to a hand-stepped session that reads `sess.logits` before and `sess.scores` after each sample(), against the oracle,
the drawn ids against the scores, tokens and waveform unchanged by asking for the outputs on every path, the B > 32 shards, the
host-driven loop, the off state, and the C ABI's window.
"""
import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg
from oracle.sampling import ParlerLogitsProcessorOracle
from tests import sampling_ext_oracle as so

DEV = "cuda"
OUT = dict(return_dict_in_generate=True, output_scores=True, output_logits=True)


# ---- host ----------------------------------------------------------------------------------------------------------------------
def test_generation_config_fields_default_off():
    from parler_tts_b200 import GenerationConfig
    gc = GenerationConfig()
    assert gc.output_scores is False and gc.output_logits is False
    assert gc.update(output_scores=True, output_logits=True) == {}
    assert gc.output_scores is True and gc.output_logits is True


def test_output_kwargs_are_known_to_generate():
    from parler_tts_b200 import GenerationConfig, ParlerTTSForConditionalGeneration
    m = ParlerTTSForConditionalGeneration.__new__(ParlerTTSForConditionalGeneration)
    m.generation_config = GenerationConfig()
    assert "output_scores" not in m._MODEL_KWARGS
    # the unknown-keyword check runs before any device work: only the misspelt name is reported
    with pytest.raises(ValueError, match=r"\['output_logit'\]"):
        m.generate(encoder_outputs=(torch.zeros(1, 2, 8),), output_scores=True, output_logits=True, output_attentions=True,
                   output_hidden_states=True, output_logit=True)


def test_window_and_chunk_arithmetic():
    from parler_tts_b200.modeling import StepOutputs, output_window, steps_in_window
    C = StepOutputs.CHUNK
    assert C == 64
    assert output_window(0, C) == (0, 0) and output_window(63, C) == (0, 0) and output_window(64, C) == (1, 64)
    assert output_window(200, C) == (3, 192)
    # from step 1 (the prefill's sample is step 0) the calls end at every chunk boundary
    calls, s, left = [], 1, 255
    while left > 0:
        n = steps_in_window(s, left, C)
        assert output_window(s, C) == output_window(s + n - 1, C)
        calls.append(n)
        s, left = s + n, left - n
    assert calls == [63, 64, 64, 64]
    assert steps_in_window(70, 3, C) == 3


def test_step_outputs_chunks_put_and_result():
    from parler_tts_b200.modeling import StepOutputs
    o = StepOutputs(rows=6, vocab_size=5, device="cpu", scores=True, logits=False)
    assert list(o.chunks) == ["scores"]
    o.put(65, 2, torch.zeros(2, 5), torch.ones(2, 5))       # chunk 1 exists from here on, chunk 0 too (NaN)
    assert len(o.chunks["scores"]) == 2
    r = o.result(66)
    assert list(r) == ["scores"] and len(r["scores"]) == 66
    assert torch.equal(r["scores"][65][2:4], torch.ones(2, 5))
    assert torch.isnan(r["scores"][65][:2]).all() and torch.isnan(r["scores"][65][4:]).all() and torch.isnan(r["scores"][3]).all()
    assert r["scores"][65].shape == (6, 5)
    assert len(o.result(130)["scores"]) == 130 and len(o.chunks["scores"]) == 3   # a result past the last chunk reads NaN


# ---- GPU helpers ---------------------------------------------------------------------------------------------------------------
def _model(cfg, seed, dtype=torch.float32, head_std=0.6, eos_bias=None):
    from oracle.weights import make_dac_weights, make_decoder_weights
    from tests.helpers import build_product_model
    w = make_decoder_weights(cfg, seed=seed, head_std=head_std)
    if eos_bias:
        for k in range(cfg.num_codebooks):
            w[f"decoder.lm_heads.{k}.weight"][cfg.eos_token_id] *= eos_bias
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=min(cfg.codebook_size, cfg.vocab_size - 8))
    return w, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=dtype)


def _kw(inputs, dtype=torch.float32):
    enc, enc_mask, prompt, prompt_mask = inputs
    return dict(encoder_outputs=(enc.to(DEV).to(dtype),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV).to(dtype),
                prompt_attention_mask=prompt_mask.to(DEV))


def _hand(model, inputs, L, gen, seed, input_ids=None, dtype=torch.float32, min_new_tokens=0):
    """The session stepped by hand: sess.logits before and sess.scores after every sample(), decode_forward() between."""
    from parler_tts_b200.modeling import GenerationConfig, resolve_sampling_ext
    enc, enc_mask, prompt, prompt_mask = inputs
    B, S, _ = enc.shape
    P = prompt.shape[1]
    n0 = 1 if input_ids is None else input_ids.shape[1]
    gc = GenerationConfig(**gen, min_new_tokens=min_new_tokens or None)
    ext, mnt = resolve_sampling_ext(gc, n0)
    sess = model.decoder.engine.session(B, P, S, P + L, max_input_len=n0)
    sess.begin(L, do_sample=gc.do_sample, temperature=gc.temperature, top_k=gc.top_k if gc.do_sample else 0, top_p=gc.top_p,
               min_new_tokens=mnt, seed=seed, ext=ext, input_ids=input_ids)
    sess.prefill(prompt.to(DEV).to(dtype), prompt_mask, enc.to(DEV).to(dtype), enc_mask)
    logits, scores = [], []
    for t in range(L - n0):
        if t > 0:
            if int(sess.state[1].item()) == 0:
                break
            sess.decode_forward()
        logits.append(sess.logits.clone())
        sess.sample()
        scores.append(sess.scores.clone())
    torch.cuda.synchronize()
    cur = int(sess.state[0].item())
    return logits, scores, sess.raw_ids[:, :cur].cpu().numpy()


def _same(a, b):
    return torch.equal(torch.nan_to_num(a, nan=7.0), torch.nan_to_num(b, nan=7.0)) and torch.equal(torch.isnan(a), torch.isnan(b))


def _check_ids_against_scores(cfg, hist, scores, n0, do_sample):
    """The greedy id of every unfinished row is the argmax of its row (lowest index on ties); a sampled id has a finite score
    unless every id was removed and the row took token 0."""
    eos = cfg.eos_token_id
    for t, s in enumerate(scores):
        s = s.cpu().numpy()
        col = n0 + t
        for r in range(hist.shape[0]):
            if (hist[r, n0:col] == eos).any():
                continue   # finished: pad from here on
            tok = hist[r, col]
            if do_sample:
                assert np.isfinite(s[r, tok]) or (tok == 0 and not np.isfinite(s[r]).any()), (t, r, tok)
            else:
                assert tok == int(np.argmax(s[r])), (t, r)


GENS = [dict(do_sample=False), dict(do_sample=True, temperature=0.8, top_k=20, top_p=0.9),
        dict(do_sample=True, top_k=0, min_p=0.05, no_repeat_ngram_size=2)]


@pytest.mark.gpu
@pytest.mark.parametrize("gen", GENS, ids=["greedy", "temp-topk-topp", "ext-minp-ngram"])
def test_tiny_fp32_outputs_match_hand_stepped_session_and_oracle(gen):
    from oracle.decoder import OracleDecoder
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    w, model = _model(cfg, seed=41)
    B, S, P, L = 3, 8, 4, 20
    inputs = synth_inputs(cfg, B, S, P, seed=5)
    out = model.generate(**_kw(inputs), max_length=L, seed=7, **gen, **OUT)
    hl, hs, hist = _hand(model, inputs, L, gen, seed=7)
    n = hist.shape[1] - 1
    assert out.raw_ids.shape[1] == hist.shape[1]
    assert len(out.scores) == len(out.logits) == n == len(hl)
    for t in range(n):
        assert out.scores[t].shape == (B * cfg.num_codebooks, cfg.vocab_size) and out.scores[t].dtype == torch.float32
        assert torch.equal(out.logits[t], hl[t]), t
        assert _same(out.scores[t], hs[t]), t
    _check_ids_against_scores(cfg, hist, out.scores, 1, gen["do_sample"])
    # the processors' oracle on the kernel's own logits and history (tolerances of test_processed_scores_match_oracle)
    parler = ParlerLogitsProcessorOracle(cfg.eos_token_id, cfg.num_codebooks, B)
    for t in range(n):
        want = so.process_scores(out.logits[t].cpu().numpy(), hist[:, :t + 1], parler, dict(gen))
        got = out.scores[t].cpu().numpy()
        kept_g, kept_w = np.isfinite(got), np.isfinite(want)
        assert (kept_g != kept_w).sum() <= 2, t
        both = kept_g & kept_w
        assert np.abs(got[both] - want[both]).max() <= 1e-5 * max(1.0, np.abs(want[both]).max()), t
    # the raw logits against the oracle decoder teacher-forced on the kernel's history
    logits_ref = []

    class Rec:
        def __init__(self, dec):
            self.dec = dec

        def prefill(self, *a):
            x = self.dec.prefill(*a)
            logits_ref.append(x[:, -1, :].float().numpy())
            return x

        def step(self, *a):
            x = self.dec.step(*a)
            logits_ref.append(x[:, -1, :].float().numpy())
            return x

    enc, enc_mask, prompt, prompt_mask = inputs
    so.generate_tokens(Rec(OracleDecoder(cfg, w, torch.float32)), cfg, enc, enc_mask, prompt, prompt_mask, dict(max_length=L),
                       pick=lambda step, s: hist[:, 1 + step])
    assert len(logits_ref) == n
    for t in range(n):
        assert np.abs(out.logits[t].cpu().numpy() - logits_ref[t]).max() < 2e-4, t


@pytest.mark.gpu
def test_continuation_outputs_cover_the_generated_columns():
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=30, head_std=0.5)
    B, S, P, L, prefix = 2, 8, 4, 24, 6
    inputs = synth_inputs(cfg, B, S, P, seed=3)
    g = np.random.default_rng(8)
    ids = np.concatenate([np.full((B * cfg.num_codebooks, 1), cfg.bos_token_id),
                          g.integers(0, 40, size=(B * cfg.num_codebooks, prefix))], axis=1).astype(np.int64)
    ids_t = torch.from_numpy(ids).to(DEV)
    n0 = ids.shape[1]
    gen = dict(do_sample=False)
    out = model.generate(**_kw(inputs), decoder_input_ids=ids_t, max_length=L, **gen, **OUT)
    assert len(out.scores) == len(out.logits) == out.raw_ids.shape[1] - n0 > 0
    hl, hs, hist = _hand(model, inputs, L, gen, seed=0, input_ids=ids_t)
    assert len(hs) == len(out.scores)
    for t in range(len(hs)):
        assert torch.equal(out.logits[t], hl[t]) and _same(out.scores[t], hs[t]), t
    _check_ids_against_scores(cfg, hist, out.scores, n0, False)


def _mini_model():
    cfg = mini_cfg(num_hidden_layers=4)
    _, model = _model(cfg, seed=21, dtype=torch.bfloat16, head_std=0.3)
    return cfg, model


@pytest.mark.gpu
def test_mini_bf16_cluster_outputs_match_hand_stepped_split_path():
    """B = 32 on the cluster kernel: generate()'s rows equal decode_forward() + sample() (the split path's own kernels), with the
    plain sampler in the hand-stepped session and the EXT sampler with every stage off in generate()."""
    from tests.helpers import synth_inputs
    cfg, model = _mini_model()
    B, L = 32, 24
    inputs = synth_inputs(cfg, B, 12, 8, seed=B)
    gen = dict(do_sample=True, top_k=50)
    out = model.generate(**_kw(inputs, torch.bfloat16), max_length=L, min_new_tokens=L, seed=11, **gen, **OUT)
    sess = model.decoder.engine._sessions[(B, 8, 12)]
    assert sess.fused == 2
    hl, hs, hist = _hand(model, inputs, L, gen, seed=11, dtype=torch.bfloat16, min_new_tokens=L)
    assert len(out.scores) == len(hs) == L - 1
    for t in range(L - 1):
        assert torch.equal(out.logits[t], hl[t]) and _same(out.scores[t], hs[t]), t
    _check_ids_against_scores(cfg, hist, out.scores, 1, True)


class _Rec:
    def __init__(self):
        self.cols = []

    def put(self, v):
        self.cols.append(v.reshape(v.shape[0], -1).clone())

    def end(self):
        pass


@pytest.mark.gpu
def test_asking_for_outputs_changes_no_token_and_no_sample(monkeypatch):
    """raw_ids and the waveform with and without both outputs: B = 32 on the cluster kernel, B = 34 in shards, PTTS_STEP=legacy,
    an EXT knob and a streamer (the streamed columns too)."""
    from tests.helpers import synth_inputs
    cfg, model = _mini_model()
    L = 40
    for B, mode, extra, streamed in [(32, None, {}, False), (34, None, {}, False), (32, "legacy", {}, False),
                                     (32, None, dict(min_p=0.05), False), (4, None, {}, True)]:
        monkeypatch.delenv("PTTS_STEP", raising=False)
        if mode:
            monkeypatch.setenv("PTTS_STEP", mode)
        inputs = synth_inputs(cfg, B, 12, 8, seed=B)
        kw = dict(**_kw(inputs, torch.bfloat16), max_length=L, min_new_tokens=L - 8, seed=11, do_sample=True, top_k=50,
                  _suppress_special=True, return_dict_in_generate=True, **extra)
        runs = []
        for outs in ({}, dict(output_scores=True, output_logits=True)):
            rec = _Rec() if streamed else None
            out = model.generate(streamer=rec, **kw, **outs)
            runs.append((out.raw_ids.cpu(), out.sequences.cpu(), None if rec is None else torch.cat(rec.cols, 1)))
            if outs:
                assert len(out.scores) == out.raw_ids.shape[1] - 1
            else:
                assert "scores" not in out and "logits" not in out
        assert torch.equal(runs[0][0], runs[1][0]), (B, mode, extra)
        assert torch.equal(runs[0][1], runs[1][1]), (B, mode, extra)
        if streamed:
            assert torch.equal(runs[0][2], runs[1][2])
    monkeypatch.delenv("PTTS_STEP", raising=False)


@pytest.mark.gpu
def test_shards_write_their_own_rows():
    """B = 34: rows of the second shard equal a B = 2 call with row_base = 32 K up to that call's length and are NaN after it;
    rows of the first shard equal a B = 32 call (NaN past its end)."""
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=7, dtype=torch.bfloat16, eos_bias=3.0)
    B, L = 34, 40
    K = cfg.num_codebooks
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, 8, 4, seed=9)
    kw = dict(do_sample=True, top_k=0, max_length=L, seed=4, **OUT)
    cut = lambda t, sl: t[sl].to(DEV)
    run = lambda sl, rb: model.generate(encoder_outputs=(cut(enc, sl).bfloat16(),), attention_mask=cut(enc_mask, sl),
                                        prompt_hidden_states=cut(prompt, sl).bfloat16(), prompt_attention_mask=cut(prompt_mask, sl),
                                        row_base=rb, **kw)
    full, a, b = run(slice(0, B), 0), run(slice(0, 32), 0), run(slice(32, B), 32 * K)
    n = len(full.scores)
    assert n == max(len(a.scores), len(b.scores)) == full.raw_ids.shape[1] - 1
    for part, lo, hi in ((a, 0, 32 * K), (b, 32 * K, B * K)):
        for t in range(n):
            got = full.scores[t][lo:hi], full.logits[t][lo:hi]
            if t < len(part.scores):
                assert _same(got[0], part.scores[t]) and torch.equal(got[1], part.logits[t]), (lo, t)
            else:
                assert torch.isnan(got[0]).all() and torch.isnan(got[1]).all(), (lo, t)
    print(f"shard lengths {len(a.scores)} / {len(b.scores)} of {n} steps")


@pytest.mark.gpu
def test_host_driven_loop_records_the_scores_after_the_callers_processor():
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=12)
    B, L = 2, 16
    inputs = synth_inputs(cfg, B, 8, 4, seed=1)
    final = []

    def proc(ids, scores):
        return scores + 0.25 * (torch.arange(scores.shape[1], device=scores.device) % 3 == 0)

    def crit(ids, scores):   # receives the scores the token was drawn from
        final.append(scores.clone())
        return torch.zeros(ids.shape[0], dtype=torch.bool, device=ids.device)

    out = model.generate(**_kw(inputs), do_sample=True, top_k=30, min_p=0.1, max_length=L, logits_processor=[proc],
                         stopping_criteria=[crit], seed=2, **OUT)
    assert len(out.scores) == len(final) == out.raw_ids.shape[1] - 1
    for t, want in enumerate(final):
        assert _same(out.scores[t], want), t
        assert torch.isfinite(out.logits[t]).all(), t


@pytest.mark.gpu
def test_off_means_off():
    """output_scores / output_logits without return_dict_in_generate: the same waveform and no output storage."""
    from tests.helpers import synth_inputs
    cfg, model = _mini_model()
    B, L = 8, 40
    inputs = synth_inputs(cfg, B, 12, 8, seed=3)
    kw = dict(**_kw(inputs, torch.bfloat16), max_length=L, seed=5, do_sample=True, top_k=50, _suppress_special=True)
    model.generate(**kw)   # warm-up: session, graphs
    peaks, waves = [], []
    for extra in ({}, dict(output_scores=True, output_logits=True)):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        w = model.generate(**kw, **extra)
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated())
        assert isinstance(w, torch.Tensor)
        waves.append(w.cpu())
        del w   # the next call's peak must not hold this one's waveform
    assert torch.equal(waves[0], waves[1])
    assert peaks[0] == peaks[1], peaks


@pytest.mark.gpu
def test_set_outputs_abi_window_and_reset():
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=41)
    B, S, P, L = 3, 8, 4, 16
    K, V = cfg.num_codebooks, cfg.vocab_size
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=5)
    sess = model.decoder.engine.session(B, P, S, P + L)
    sess.begin(L, do_sample=True, top_k=20, seed=3, min_new_tokens=L)
    rows = B * K
    buf = torch.full((2, 7, rows + 1, V), -12345.0, device=DEV)   # slots 0 and 6 lie outside the window; row `rows` is the gap
    with pytest.raises(ValueError):
        sess.set_outputs(buf[0, 1, 0], buf[1, 1, 0], 3, 5, rows * V - 1)
    with pytest.raises(ValueError):
        sess.set_outputs(buf[0, 1, 0], buf[1, 1, 0], 3, -1, (rows + 1) * V)
    sess.set_outputs(buf[0, 1, 0], buf[1, 1, 0], 3, 5, (rows + 1) * V)   # steps 3 .. 7
    sess.prefill(prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
    logits, scores = [], []
    for t in range(L - 1):
        if t > 0:
            sess.decode_forward()
        logits.append(sess.logits.clone())
        sess.sample()
        scores.append(sess.scores.clone())
    torch.cuda.synchronize()
    for i, t in enumerate(range(3, 8)):
        assert torch.equal(buf[0, 1 + i, :rows], logits[t]) and _same(buf[1, 1 + i, :rows], scores[t]), t
    outside = torch.ones(7, rows + 1, dtype=torch.bool, device=DEV)
    outside[1:6, :rows] = False
    assert (buf[:, outside] == -12345.0).all()
    # a new generation starts with the outputs off: the old buffers stay as they are
    before = buf.clone()
    sess.begin(L, do_sample=True, top_k=20, seed=4, min_new_tokens=L)
    sess.prefill(prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
    sess.sample()
    sess.decode_steps(L - 2)
    torch.cuda.synchronize()
    assert torch.equal(buf, before)
