"""generate()'s further processors: no_repeat_ngram_size, min_length, min_p, typical_p, epsilon_cutoff and eta_cutoff.

Host tests: the CPU oracle (tests/sampling_ext_oracle.py) against tests/golden/sampling_ext.npz (transformers' classes executed),
and generate()'s validation against what transformers raises.  GPU tests: the EXT sampler's processed scores and draws against
the oracle, greedy free-running runs token for token, and the split path (step kernel without its sampling phase + EXT sampler)
bit-identical to the default path when no stage changes anything.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg
from oracle.sampling import ParlerLogitsProcessorOracle, softmax_rows
from tests import sampling_ext_oracle as so

DEV = "cuda"


# ---- host: the oracle and the validation against the executed library ----------------------------------------------------------
@pytest.fixture(scope="module")
def fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "sampling_ext.npz"))


def test_oracle_processors_match_fixture(fixture):
    z = fixture
    scores, ids = z["scores"], z["ids"]
    fns = {"ngram": lambda s, v: so.no_repeat_ngram(ids, s, int(v)), "min_p": so.min_p, "typical": so.typical,
           "epsilon": so.epsilon, "eta": so.eta}
    for name, fn in fns.items():
        for i, v in enumerate(z[f"{name}_values"]):
            got = fn(scores.copy(), float(v))
            assert np.array_equal(got, z[f"{name}_{i}"]), (name, v)


def test_oracle_chain_and_order_match_fixture(fixture):
    z = fixture
    names = {"no_repeat_ngram_size": "NoRepeatNGramLogitsProcessor", "min_length": "MinLengthLogitsProcessor",
             "min_new_tokens": "MinNewTokensLengthLogitsProcessor", "temperature": "TemperatureLogitsWarper",
             "top_k": "TopKLogitsWarper", "top_p": "TopPLogitsWarper", "min_p": "MinPLogitsWarper",
             "typical_p": "TypicalLogitsWarper", "epsilon_cutoff": "EpsilonLogitsWarper", "eta_cutoff": "EtaLogitsWarper"}
    order = ["no_repeat_ngram_size", "min_length", "min_new_tokens", "parler", "temperature", "top_k", "top_p", "min_p", "typical_p",
             "epsilon_cutoff", "eta_cutoff"]
    ci = 0
    while f"chain{ci}_out" in z:
        knobs = json.loads(str(z[f"chain{ci}_knobs"]))
        want = [names.get(k, "ParlerTTSLogitsProcessor") for k in order
                if k == "parler" or (k in knobs and (knobs.get("do_sample") or k in ("no_repeat_ngram_size", "min_length", "min_new_tokens")))]
        assert json.loads(str(z[f"chain{ci}_order"])) == want, ci
        gen = dict(knobs)
        parler = ParlerLogitsProcessorOracle(1024, 3, 2)
        # the fixture's history has 40 columns and no decoder input beyond the BOS column: n0 = 1
        got = so.process_scores(z["scores"], z["ids"], parler, gen, n0=1)
        assert np.array_equal(got, z[f"chain{ci}_out"]), ci
        ci += 1
    assert ci == 6


def test_generate_validation_matches_transformers(fixture):
    from parler_tts_b200 import GenerationConfig
    from parler_tts_b200.modeling import resolve_sampling_ext
    for knob, value, status in json.loads(str(fixture["validation"])):
        gc = GenerationConfig(do_sample=True, top_k=0, **{knob: value})
        if status == 2:
            with pytest.raises(ValueError):
                resolve_sampling_ext(gc, 1)
            continue
        ext, mnt = resolve_sampling_ext(gc, 1)
        on = ext is not None or mnt > 0
        if knob == "min_p" and value == 0.0:
            on = True   # transformers builds a MinP warper that removes nothing; the device loop leaves it off
            assert ext is None
            continue
        assert on == (status == 1), (knob, value)
    # greedy: the warpers are not built, so they neither raise nor act
    assert resolve_sampling_ext(GenerationConfig(do_sample=False, min_p=1.5, typical_p=0.0, eta_cutoff=0.5), 1) == (None, 0)


def test_min_length_fold_matches_transformers(fixture):
    from parler_tts_b200 import GenerationConfig
    from parler_tts_b200.modeling import resolve_sampling_ext
    for ml, mnt, n0, folded in json.loads(str(fixture["fold"])):
        gc = GenerationConfig(do_sample=False, min_length=0 if ml is None else ml, min_new_tokens=mnt)
        _, got = resolve_sampling_ext(gc, n0)
        want = max(0, (folded or 0) - n0)
        assert got == want, (ml, mnt, n0)
        assert got == so.folded_min_new_tokens(ml, mnt, n0)


def test_repetition_penalty_still_rejected():
    from parler_tts_b200 import ParlerTTSConfig, ParlerTTSForConditionalGeneration  # noqa: F401
    from parler_tts_b200 import GenerationConfig
    m = ParlerTTSForConditionalGeneration.__new__(ParlerTTSForConditionalGeneration)
    m.generation_config = GenerationConfig()
    with pytest.raises(ValueError, match="repetition_penalty"):
        m.generate(encoder_outputs=(torch.zeros(1, 2, 8),), repetition_penalty=1.3)


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
def _model(cfg, seed, dtype=torch.float32, head_std=0.6, eos_bias=None):
    from oracle.weights import make_dac_weights, make_decoder_weights
    from tests.helpers import build_product_model
    w = make_decoder_weights(cfg, seed=seed, head_std=head_std)
    if eos_bias:
        for k in range(cfg.num_codebooks):
            w[f"decoder.lm_heads.{k}.weight"][cfg.eos_token_id] *= eos_bias
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=min(cfg.codebook_size, cfg.vocab_size - 8))
    return w, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=dtype)


EXT_KNOBS = [dict(min_p=0.1), dict(typical_p=0.7), dict(epsilon_cutoff=0.01), dict(eta_cutoff=0.005), dict(no_repeat_ngram_size=2),
             dict(no_repeat_ngram_size=1, min_p=0.05),
             dict(temperature=0.8, top_k=40, top_p=0.95, min_p=0.02, typical_p=0.9, epsilon_cutoff=3e-4, eta_cutoff=3e-4,
                  no_repeat_ngram_size=3)]


@pytest.mark.gpu
@pytest.mark.parametrize("V,dtype", [(96, torch.float32), (1088, torch.bfloat16)], ids=["fp32-V96", "bf16-V1088"])
@pytest.mark.parametrize("knobs", EXT_KNOBS, ids=lambda k: "+".join(sorted(k)))
def test_processed_scores_match_oracle(V, dtype, knobs):
    """sess.scores after every sample() == the oracle chain on the kernel's own logits and history: same kept set up to ids at a
    warper's threshold, equal values where both keep, every draw inside the kept set."""
    from parler_tts_b200.modeling import GenerationConfig, resolve_sampling_ext
    cfg = tiny_cfg(vocab_size=V)
    _, model = _model(cfg, seed=41, dtype=dtype)
    from tests.helpers import synth_inputs
    B, S, P, L = 3, 8, 4, 14
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=5)
    gen = {"do_sample": True, "top_k": 0, **knobs}
    ext, _ = resolve_sampling_ext(GenerationConfig(**gen), 1)
    sess = model.decoder.engine.session(B, P, S, P + L)
    sess.begin(L, seed=7, do_sample=True, temperature=gen.get("temperature", 1.0), top_k=gen["top_k"], top_p=gen.get("top_p", 1.0),
               ext=ext)
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
        want = so.process_scores(logits, raw, parler, dict(gen))
        kept_g, kept_w = np.isfinite(got), np.isfinite(want)
        # a threshold decision may flip for an id whose tested quantity lies at the threshold (different summation order)
        assert (kept_g != kept_w).sum() <= 2, (t, (kept_g != kept_w).sum())
        both = kept_g & kept_w
        assert np.abs(got[both] - want[both]).max() <= 1e-5 * max(1.0, np.abs(want[both]).max())
        tok = sess.raw_ids[:, t + 1].cpu().numpy()
        for r in range(tok.shape[0]):
            assert kept_g[r, tok[r]] or tok[r] == cfg.pad_token_id or not kept_g[r].any(), (t, r)


@pytest.mark.gpu
@pytest.mark.parametrize("knobs", [dict(typical_p=0.6), dict(min_p=0.15)], ids=["typical", "min_p"])
def test_sampling_distribution(knobs):
    """The EXT sampler's draws follow its processed distribution (chi-square over many seeds)."""
    from parler_tts_b200.modeling import GenerationConfig, resolve_sampling_ext
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=43, head_std=0.15)
    B, S, P, L = 2, 6, 3, 4
    enc, _, prompt, _ = synth_inputs(cfg, B, S, P, seed=6, masks=False)
    ext, _ = resolve_sampling_ext(GenerationConfig(do_sample=True, **knobs), 1)
    sess = model.decoder.engine.session(B, P, S, P + L)
    counts, probs, N = None, None, 600
    for seed in range(N):
        sess.begin(L, do_sample=True, seed=seed, ext=ext)
        sess.prefill(prompt.to(DEV), None, enc.to(DEV), None)
        sess.sample()
        tok = sess.raw_ids[:, 1].cpu().numpy()
        if counts is None:
            probs = softmax_rows(sess.scores.cpu().numpy())
            counts = np.zeros_like(probs)
        counts[np.arange(tok.shape[0]), tok] += 1
    kept = (probs > 0).sum(1)
    assert ((kept > 1) & (kept < cfg.vocab_size)).any(), kept   # the warper removed some ids and kept several
    for r in range(counts.shape[0]):
        nz = probs[r] > 0
        assert counts[r][~nz].sum() == 0
        exp = probs[r][nz] * N
        chi2 = ((counts[r][nz] - exp) ** 2 / np.maximum(exp, 1e-9)).sum()
        dof = nz.sum() - 1
        assert chi2 < dof + 6 * np.sqrt(2 * dof) + 10, (r, chi2, dof)


def _greedy_session(model, cfg, inputs, L, ext, mnt=0, input_ids=None):
    enc, enc_mask, prompt, prompt_mask = inputs
    B, S, _ = enc.shape
    P = prompt.shape[1]
    n0 = 1 if input_ids is None else input_ids.shape[1]
    sess = model.decoder.engine.session(B, P, S, P + L, max_input_len=n0)
    sess.begin(L, do_sample=False, min_new_tokens=mnt, ext=ext, input_ids=input_ids)
    sess.prefill(prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
    sess.sample()
    sess.decode_steps(L - n0 - 1)
    torch.cuda.synchronize()
    return int(sess.state[0].item()), sess.raw_ids.cpu().numpy()


def _margins_ok(scores):
    fin = [np.sort(np.where(np.isfinite(s), s, -1e30), -1) for s in scores]
    return min(float((f[:, -1] - f[:, -2]).min()) for f in fin)


@pytest.mark.gpu
@pytest.mark.parametrize("n,prefix", [(2, 0), (3, 0), (2, 6)], ids=["n2", "n3", "n2-prefix6"])
def test_greedy_no_repeat_ngram_matches_oracle(n, prefix):
    """fp32 tiny, greedy with n-gram bans (the prefix's n-grams count when continuing): token for token."""
    from oracle.decoder import OracleDecoder
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    w, model = _model(cfg, seed=30, head_std=0.5)   # seed chosen so the oracle's smallest top-2 margin is >= 1.3e-3 in every case
    B, S, P, L = 4, 8, 4, 40
    inputs = synth_inputs(cfg, B, S, P, seed=3)
    enc, enc_mask, prompt, prompt_mask = inputs
    dec_ids = None
    if prefix:
        g = np.random.default_rng(8)
        dec_ids = g.integers(0, 40, size=(B * cfg.num_codebooks, prefix)).astype(np.int64)
        dec_ids[:, 2:4] = dec_ids[:, 4:6]   # planted repeats inside the prefix
    ref = so.generate_tokens(OracleDecoder(cfg, w, torch.float32), cfg, enc, enc_mask, prompt, prompt_mask,
                             dict(max_length=L, do_sample=False, no_repeat_ngram_size=n), decoder_input_ids=dec_ids)
    assert _margins_ok(ref["scores"]) > 1e-3, "test weights give near-ties; pick another seed"
    ids = None if dec_ids is None else torch.from_numpy(ref["input_ids"]).to(DEV)
    ext = dict(no_repeat_ngram_size=n, min_p=0.0, typical_p=1.0, epsilon_cutoff=0.0, eta_cutoff=0.0)
    cur, raw = _greedy_session(model, cfg, inputs, L, ext, input_ids=ids)
    m = ref["raw_ids"].shape[1]
    assert cur == m
    assert np.array_equal(raw[:, :m], ref["raw_ids"])
    plain_cur, plain = _greedy_session(model, cfg, inputs, L, None, input_ids=ids)
    assert not np.array_equal(plain[:, :plain_cur], ref["raw_ids"]), "the bans should change this run"


@pytest.mark.gpu
def test_min_length_equals_min_new_tokens_and_oracle():
    """EOS-biased heads: generate(min_length=m) gives no EOS before column m, equals generate(min_new_tokens=m - n0), and matches the
    oracle's MinLength loop token for token."""
    from oracle.decoder import OracleDecoder
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    w, model = _model(cfg, seed=31, head_std=0.5, eos_bias=6.0)
    B, S, P, L, ml = 4, 8, 4, 48, 20
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=4)
    kw = dict(encoder_outputs=(enc.to(DEV),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV),
              prompt_attention_mask=prompt_mask.to(DEV), do_sample=False, max_length=L, return_codes=True)
    _, a = model.generate(min_length=ml, **kw)
    _, b = model.generate(min_new_tokens=ml - 1, **kw)
    _, c = model.generate(**kw)
    assert torch.equal(a.raw_ids, b.raw_ids)
    ra = a.raw_ids.cpu().numpy()
    assert not (ra[:, :ml] == cfg.eos_token_id).any()
    assert (c.raw_ids.cpu().numpy()[:, :ml] == cfg.eos_token_id).any(), "the heads should want EOS early"
    ref = so.generate_tokens(OracleDecoder(cfg, w, torch.float32), cfg, enc, enc_mask, prompt, prompt_mask,
                             dict(max_length=L, do_sample=False, min_length=ml))
    assert _margins_ok(ref["scores"]) > 1e-3
    cur, raw = _greedy_session(model, cfg, (enc, enc_mask, prompt, prompt_mask), L, None, mnt=ml - 1)
    assert np.array_equal(raw[:, :ref["raw_ids"].shape[1]], ref["raw_ids"])


@pytest.mark.gpu
def test_ngram_one_sampled_ends_inside_the_vocabulary():
    """n = 1 bans every id seen: with EOS masked, rows run out of candidates on V = 96 after 94 draws, take token 0 from then on,
    and the call still ends."""
    from tests.helpers import synth_inputs
    cfg = tiny_cfg(max_position_embeddings=256)
    _, model = _model(cfg, seed=5)
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, 2, 8, 4, seed=2)
    L = 200
    _, out = model.generate(encoder_outputs=(enc.to(DEV),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV),
                            prompt_attention_mask=prompt_mask.to(DEV), do_sample=True, top_k=0, no_repeat_ngram_size=1,
                            max_length=L, min_new_tokens=L, return_codes=True, seed=3)
    raw = out.raw_ids.cpu().numpy()
    assert raw.shape[1] == L
    assert raw.min() >= 0 and raw.max() < cfg.vocab_size
    assert (raw[:, 120:L - cfg.num_codebooks] == 0).all()


def _mini_model():
    cfg = mini_cfg(num_hidden_layers=4)
    _, model = _model(cfg, seed=21, dtype=torch.bfloat16, head_std=0.3)
    return cfg, model


class _Rec:
    def __init__(self):
        self.cols = []

    def put(self, v):
        self.cols.append(v.reshape(v.shape[0], -1).clone())

    def end(self):
        pass


@pytest.mark.gpu
@pytest.mark.parametrize("gen", [dict(do_sample=False), dict(do_sample=True, top_k=50)], ids=["greedy", "topk50"])
def test_split_path_is_bit_identical_to_the_default_path(monkeypatch, gen):
    """no_repeat_ngram_size = max_length + 1 bans nothing but runs every token as step kernel + EXT sampler: the ids equal the
    default path's bit for bit (B = 32 on the cluster kernel, B = 34 in shards, PTTS_STEP=legacy, a streamer)."""
    from tests.helpers import synth_inputs
    cfg, model = _mini_model()
    L = 40
    for B, mode, streamed in [(32, None, False), (34, None, False), (32, "legacy", False), (4, None, True)]:
        monkeypatch.delenv("PTTS_STEP", raising=False)
        if mode:
            monkeypatch.setenv("PTTS_STEP", mode)
        enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, 12, 8, seed=B)
        kw = dict(encoder_outputs=(enc.to(DEV).bfloat16(),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV).bfloat16(),
                  prompt_attention_mask=prompt_mask.to(DEV), max_length=L, min_new_tokens=L, return_codes=True, seed=11,
                  _suppress_special=True, **gen)
        runs = []
        for extra in ({}, dict(no_repeat_ngram_size=L + 1)):
            rec = _Rec() if streamed else None
            _, out = model.generate(streamer=rec, **kw, **extra)
            runs.append((out.raw_ids.cpu(), None if rec is None else torch.cat(rec.cols, 1)))
        assert torch.equal(runs[0][0], runs[1][0]), (B, mode)
        if streamed:
            assert torch.equal(runs[0][1], runs[1][1])
    monkeypatch.delenv("PTTS_STEP", raising=False)


@pytest.mark.gpu
def test_typical_sampling_is_shard_invariant():
    """B = 34 runs as shards of 32 + 2; each utterance's draws depend on (seed, global row, column) only."""
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=7, dtype=torch.bfloat16)
    B, L = 34, 30
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, 8, 4, seed=9)
    kw = dict(do_sample=True, top_k=0, typical_p=0.8, no_repeat_ngram_size=3, max_length=L, return_codes=True, seed=4)
    cut = lambda t, sl: t[sl].to(DEV)
    run = lambda sl, rb: model.generate(encoder_outputs=(cut(enc, sl).bfloat16(),), attention_mask=cut(enc_mask, sl),
                                        prompt_hidden_states=cut(prompt, sl).bfloat16(), prompt_attention_mask=cut(prompt_mask, sl),
                                        row_base=rb, **kw)[1].raw_ids.cpu()
    full = run(slice(0, B), 0)
    a, b = run(slice(0, 32), 0), run(slice(32, B), 32 * cfg.num_codebooks)
    n = full.shape[1]
    pad = lambda t: torch.nn.functional.pad(t, (0, n - t.shape[1]), value=cfg.pad_token_id)
    assert torch.equal(full, torch.cat([pad(a), pad(b)], 0))


@pytest.mark.gpu
def test_caller_processor_with_min_p_and_ngram_matches_oracle():
    """The host-driven loop (a caller's logits_processor): bans before the EOS masks, min_p after top-k, as the oracle orders them."""
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=12)
    B, L = 2, 16
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, 8, 4, seed=1)
    seen, final = [], []

    def proc(ids, scores):
        seen.append((ids.cpu().numpy().copy(), scores.cpu().numpy().copy()))
        return scores

    def crit(ids, scores):
        final.append((ids.cpu().numpy().copy(), scores.cpu().numpy().copy()))
        return torch.zeros(ids.shape[0], dtype=torch.bool, device=ids.device)

    model.generate(encoder_outputs=(enc.to(DEV),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV),
                   prompt_attention_mask=prompt_mask.to(DEV), do_sample=True, top_k=30, min_p=0.1, no_repeat_ngram_size=2,
                   max_length=L, logits_processor=[proc], stopping_criteria=[crit], seed=2)
    assert len(seen) == len(final) > 3
    for (ids, s_in), (ids_after, s_out) in zip(seen, final):
        banned = so.no_repeat_ngram(ids, np.zeros_like(s_in), 2)
        assert np.all(np.isneginf(s_in[np.isneginf(banned)])), "banned ids must reach the caller's processor at -inf"
        want = so.min_p(so.top_k(s_in, 30), 0.1)
        assert np.array_equal(np.isfinite(s_out), np.isfinite(want))
        tok = ids_after[:, -1]
        assert all(np.isfinite(s_out[r, tok[r]]) or tok[r] == cfg.pad_token_id for r in range(len(tok)))
