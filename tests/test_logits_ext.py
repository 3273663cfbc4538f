"""generate()'s remaining logits processors: sequence_bias, suppress_tokens, begin_suppress_tokens, exponential_decay_length_penalty,
forced_bos_token_id, forced_eos_token_id, remove_invalid_values and renormalize_logits.

Host tests: the CPU oracle (tests/logits_ext_oracle.py) and the host-driven loop's torch ops against tests/golden/logits_ext.npz
(transformers' classes and _get_logits_processor executed), and resolve_logits_ext's validation against what transformers raises.
GPU tests: the EXT sampler's processed scores against the oracle on the session's own logits, greedy runs token for token, the
decay's effect on lengths, renormalize_logits' draw rule, the split path bit-identical to the default path when no stage changes
anything, and the routes of generate() (shards, num_return_sequences, continuation, the host-driven loop).
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg
from oracle.sampling import ParlerLogitsProcessorOracle
from tests import logits_ext_oracle as lo

DEV = "cuda"
EOS = 1024
# renormalize_logits: the device's log_softmax sums in its own order; |device - torch| <= this * max(1, |score|)
LOG_SOFTMAX_TOL = 4e-6


# ---- host ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "logits_ext.npz"))


def _knobs(z, key):
    kw = json.loads(str(z[key]))
    if "exponential_decay_length_penalty" in kw:
        kw["exponential_decay_length_penalty"] = tuple(kw["exponential_decay_length_penalty"])
    return kw


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_oracle_processors_match_fixture(fixture):
    z = fixture
    scores, ids = z["scores"], z["ids"]
    n = 0
    for key in sorted(k for k in z.files if k.endswith("_knobs") and not k.startswith("chain")):
        name, i = key[:-len("_knobs")].rsplit("_", 1)
        kw = _knobs(z, key)
        h = ids[:, :kw.get("cols", ids.shape[1])]
        if name == "seq_bias":
            got = lo.sequence_bias(h, scores, kw["sequence_bias"])
        elif name == "suppress":
            got = lo.suppress(scores, kw["suppress_tokens"])
        elif name == "begin_suppress":
            got = lo.begin_suppress(h, scores, kw["begin_suppress_tokens"], kw["begin_index"])
        elif name == "decay":
            start, factor = kw["exponential_decay_length_penalty"]
            got = lo.exponential_decay(h, scores, start, factor, kw["n0"], EOS)
        elif name == "forced_bos":
            got = lo.forced(scores, kw["forced_bos_token_id"]) if h.shape[1] == 1 else scores
        elif name == "forced_eos":
            got = lo.forced(scores, kw["forced_eos_token_id"]) if h.shape[1] == kw["max_length"] - 1 else scores
        elif name == "infnan":
            got = lo.infnan(scores)
        else:
            got = lo.log_softmax(scores)
        assert _same(got, z[f"{name}_{i}"]), key
        n += 1
    assert n == 15


_NAMES = {"sequence_bias": "SequenceBiasLogitsProcessor", "no_repeat_ngram_size": "NoRepeatNGramLogitsProcessor",
          "min_new_tokens": "MinNewTokensLengthLogitsProcessor", "forced_bos_token_id": "ForcedBOSTokenLogitsProcessor",
          "forced_eos_token_id": "ForcedEOSTokenLogitsProcessor", "remove_invalid_values": "InfNanRemoveLogitsProcessor",
          "exponential_decay_length_penalty": "ExponentialDecayLengthPenalty", "suppress_tokens": "SuppressTokensLogitsProcessor",
          "begin_suppress_tokens": "SuppressTokensAtBeginLogitsProcessor", "parler": "ParlerTTSLogitsProcessor",
          "temperature": "TemperatureLogitsWarper", "top_k": "TopKLogitsWarper", "top_p": "TopPLogitsWarper",
          "min_p": "MinPLogitsWarper", "renormalize_logits": "LogitNormalization"}
_ORDER = ["sequence_bias", "no_repeat_ngram_size", "min_new_tokens", "forced_bos_token_id", "forced_eos_token_id",
          "remove_invalid_values", "exponential_decay_length_penalty", "suppress_tokens", "begin_suppress_tokens", "parler",
          "temperature", "top_k", "top_p", "min_p", "renormalize_logits"]


def _chains(z):
    ci = 0
    while f"chain{ci}_out" in z:
        cols, n0 = (int(v) for v in z[f"chain{ci}_cols_n0"])
        yield ci, _knobs(z, f"chain{ci}_knobs"), cols, n0
        ci += 1


def test_oracle_chain_and_order_match_fixture(fixture):
    """Every chain bit for bit, and the class order the oracle assumes is the one _get_logits_processor builds."""
    z = fixture
    n = 0
    for ci, knobs, cols, n0 in _chains(z):
        sampling = {"temperature", "top_k", "top_p", "min_p"}
        want = [_NAMES[k] for k in _ORDER if k == "parler" or (k in knobs and knobs[k] not in (0, None)
                                                              and (knobs.get("do_sample") or k not in sampling))]
        assert json.loads(str(z[f"chain{ci}_order"])) == want, ci
        parler = ParlerLogitsProcessorOracle(EOS, 3, 2)
        got = lo.process_scores(z["scores"], z["ids"][:, :cols], parler, dict(knobs), n0=n0, max_length=knobs.get("max_length", 20))
        assert _same(got, z[f"chain{ci}_out"]), ci
        n += 1
    assert n == 8


def test_host_loop_stages_match_fixture(fixture):
    """The host-driven loop's torch ops (LogitsExt) on the fixture's chains without the warpers: bit for bit."""
    from parler_tts_b200 import GenerationConfig
    from parler_tts_b200.modeling import no_repeat_ngram_mask, resolve_logits_ext
    z = fixture
    for ci, knobs, cols, n0 in _chains(z):
        if knobs.get("do_sample"):
            continue
        L = knobs.get("max_length", 100)
        lx = resolve_logits_ext(GenerationConfig(**knobs), n0, L, 1088, EOS)
        ids = torch.from_numpy(z["ids"][:, :cols])
        s = lx.sequence_bias(ids, torch.from_numpy(z["scores"]).clone())
        s = no_repeat_ngram_mask(ids, s, int(knobs.get("no_repeat_ngram_size") or 0))
        mnt = knobs.get("min_new_tokens") or 0
        if cols - n0 < mnt:
            s[:, EOS] = -float("inf")
        s = lx.before_parler(ids, s).numpy()
        s = ParlerLogitsProcessorOracle(EOS, 3, 2)(ids.numpy(), s)
        s = lx.normalize(torch.from_numpy(np.ascontiguousarray(s))).numpy()
        assert _same(s, z[f"chain{ci}_out"]), ci


def _gc_from_record(knob):
    from parler_tts_b200 import GenerationConfig
    if "sequence_bias_dict" in knob:
        sb = {}
        for k, v, as_tuple in knob["sequence_bias_dict"]:
            sb[tuple(k) if as_tuple else k[0]] = v
        knob = dict(sequence_bias=sb)
    elif "sequence_bias_list" in knob:
        knob = dict(sequence_bias=[[tuple(k) if as_tuple else k, v] for k, v, as_tuple in knob["sequence_bias_list"]])
    return GenerationConfig(do_sample=False, **knob)


def test_resolver_raises_where_transformers_raises(fixture):
    """status 2 (transformers raises, when it builds the list or at its first call) <=> ValueError up front; an accepted knob is
    on unless it changes nothing (off values, an empty suppress list).  Beyond transformers: a forced id >= V raises up front even
    where transformers' processor never reaches the column that would index it."""
    from parler_tts_b200.modeling import resolve_logits_ext
    for knob, status, _exc in json.loads(str(fixture["validation"])):
        gc = _gc_from_record(knob)
        forced_oov = any(knob.get(k) is not None and knob[k] >= 1088 for k in ("forced_bos_token_id", "forced_eos_token_id"))
        if status == 2 or forced_oov:
            with pytest.raises(ValueError):
                resolve_logits_ext(gc, 1, 41, 1088, EOS)
            continue
        lx = resolve_logits_ext(gc, 1, 41, 1088, EOS)
        noop = knob in ({"suppress_tokens": []}, {"suppress_tokens": [1091]})
        assert (lx is not None) == (status == 1 and not noop), knob
    # the list and dict forms give the same tables, in order
    from parler_tts_b200 import GenerationConfig
    a = resolve_logits_ext(GenerationConfig(sequence_bias={(3, 7): -2.0, (7,): 1.5, (5, 9, 7): 0.75}), 1, 50, 1088, EOS)
    b = resolve_logits_ext(GenerationConfig(sequence_bias=[[[3, 7], -2.0], [[7], 1.5], [[5, 9, 7], 0.75]]), 1, 50, 1088, EOS)
    assert a.seqs == b.seqs == [((3, 7), -2.0), ((5, 9, 7), 0.75)] and np.array_equal(a.bias1, b.bias1)
    # the device loop's caps
    with pytest.raises(ValueError, match="sequence_bias"):
        resolve_logits_ext(GenerationConfig(sequence_bias={tuple(range(1, 18)): 1.0}), 1, 50, 1088, EOS)
    with pytest.raises(ValueError, match="sequence_bias"):
        resolve_logits_ext(GenerationConfig(sequence_bias={(i, 7): 1.0 for i in range(65)}), 1, 50, 1088, EOS)
    assert resolve_logits_ext(GenerationConfig(sequence_bias={(i, 7): 1.0 for i in range(64)}), 1, 50, 1088, EOS) is not None
    with pytest.raises(ValueError, match="forced_eos_token_id"):
        resolve_logits_ext(GenerationConfig(forced_eos_token_id=[5, 6]), 1, 50, 1088, EOS)
    assert resolve_logits_ext(GenerationConfig(), 1, 50, 1088, EOS) is None


def test_begin_index_and_regulation_start():
    from parler_tts_b200 import GenerationConfig
    from parler_tts_b200.modeling import resolve_logits_ext
    for n0, fb, want in [(1, None, 1), (1, 9, 2), (5, None, 5), (5, 9, 5)]:
        lx = resolve_logits_ext(GenerationConfig(begin_suppress_tokens=[3], forced_bos_token_id=fb), n0, 60, 1088, EOS)
        assert lx.begin_index == want == lo.begin_index(n0, fb)
    for n0 in (1, 7):
        lx = resolve_logits_ext(GenerationConfig(exponential_decay_length_penalty=(12, 1.1)), n0, 60, 1088, EOS)
        assert lx.decay_start == 12 + n0


def test_decay_table_is_python_pow_rounded_once():
    from parler_tts_b200 import GenerationConfig
    from parler_tts_b200.modeling import resolve_logits_ext
    for start, factor, n0, L in [(10, 1.2, 1, 200), (3, 0.97, 4, 90), (0, 3.7, 2, 50), (40, 1.5, 1, 30)]:
        lx = resolve_logits_ext(GenerationConfig(exponential_decay_length_penalty=(start, factor)), n0, L, 1088, EOS)
        want = np.zeros(L, dtype=np.float32)
        for c in range(start + n0 + 1, L):
            want[c] = np.float32(pow(factor, c - (start + n0)) - 1)
        assert _same(lx.decay, want)
        assert _same(lx.decay, lo.decay_table(start, factor, n0, L))


def test_unknown_knobs_still_rejected():
    from parler_tts_b200 import GenerationConfig, ParlerTTSForConditionalGeneration
    m = ParlerTTSForConditionalGeneration.__new__(ParlerTTSForConditionalGeneration)
    m.generation_config = GenerationConfig()
    for kw in (dict(repetition_penalty=1.3), dict(bad_words_ids=[[5]]), dict(guidance_scale=3.0)):
        with pytest.raises(ValueError, match=next(iter(kw))):
            m.generate(encoder_outputs=(torch.zeros(1, 2, 8),), suppress_tokens=[5], **kw)


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
def _model(cfg, seed, dtype=torch.float32, head_std=0.6):
    from oracle.weights import make_dac_weights, make_decoder_weights
    from tests.helpers import build_product_model
    w = make_decoder_weights(cfg, seed=seed, head_std=head_std)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=min(cfg.codebook_size, cfg.vocab_size - 8))
    return w, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=dtype)


def _compare(got, want, gen, t):
    """Bit for bit without renormalize_logits; with it, the same -inf / NaN pattern and values within LOG_SOFTMAX_TOL."""
    if not gen.get("renormalize_logits"):
        assert _same(got, want), (t, np.argwhere(got.view(np.uint32) != want.view(np.uint32))[:5])
        return
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isneginf(got), np.isneginf(want)), t
    fin = np.isfinite(want)
    assert np.all(np.abs(got[fin] - want[fin]) <= LOG_SOFTMAX_TOL * np.maximum(1.0, np.abs(want[fin]))), t


SESSION_KNOBS = [
    dict(do_sample=False, sequence_bias={(3, 7): -2.0, (7,): 1.5, (5, 7): 0.75, (7, 7): 4.0, (11,): -3.0}, suppress_tokens=[0, 9],
         begin_suppress_tokens=[1, 2, 3], forced_eos_token_id=4),
    dict(do_sample=False, remove_invalid_values=True, exponential_decay_length_penalty=(3, 1.4), suppress_tokens=[5],
         min_new_tokens=6, forced_bos_token_id=8),
    dict(do_sample=True, top_k=20, temperature=0.9, sequence_bias={(2,): 0.5, (4, 6): 1.0}, exponential_decay_length_penalty=(2, 1.2),
         renormalize_logits=True),
    dict(do_sample=False, renormalize_logits=True, suppress_tokens=[1], remove_invalid_values=True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("V,dtype", [(96, torch.float32), (1088, torch.bfloat16)], ids=["fp32-V96", "bf16-V1088"])
@pytest.mark.parametrize("knobs", SESSION_KNOBS, ids=["bias+suppress+forced_eos", "infnan+decay+forced_bos", "sampled+renorm",
                                                      "greedy+renorm"])
def test_processed_scores_match_oracle(V, dtype, knobs):
    """sess.scores after every sample() == the oracle chain on the kernel's own logits and history (greedy: bit for bit; sampled
    rows: the warpers' kept set up to 2 threshold flips, equal values where both keep)."""
    from parler_tts_b200.modeling import GenerationConfig, resolve_logits_ext, resolve_sampling_ext
    from tests.helpers import synth_inputs
    cfg = tiny_cfg(vocab_size=V)
    _, model = _model(cfg, seed=41, dtype=dtype)
    B, S, P, L = 3, 8, 4, 14
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=5)
    gen = dict(knobs)
    gc = GenerationConfig(**gen)
    ext, mnt = resolve_sampling_ext(gc, 1)
    lext = resolve_logits_ext(gc, 1, L, V, cfg.eos_token_id)
    sess = model.decoder.engine.session(B, P, S, P + L)
    sess.begin(L, seed=7, do_sample=gen["do_sample"], temperature=gen.get("temperature", 1.0), top_k=gen.get("top_k", 0),
               min_new_tokens=mnt, ext=ext, lext=lext)
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
        want = lo.process_scores(logits, raw, parler, gen, 1, L)
        if gen["do_sample"] and gen.get("top_k"):
            kept_g, kept_w = np.isfinite(got), np.isfinite(want)
            assert (kept_g != kept_w).sum() <= 2, t
            both = kept_g & kept_w
            assert np.all(np.abs(got[both] - want[both]) <= LOG_SOFTMAX_TOL * np.maximum(1.0, np.abs(want[both]))), t
        else:
            _compare(got, want, gen, t)
        if int(sess.state[1].item()) == 0:
            break


@pytest.mark.gpu
def test_generate_scores_mini_bf16_b32_match_oracle():
    """The issue's call on Mini bf16, B = 32: output_scores equal the oracle applied to output_logits and the recorded history."""
    from tests.helpers import synth_inputs
    cfg = mini_cfg(num_hidden_layers=4)
    _, model = _model(cfg, seed=21, dtype=torch.bfloat16, head_std=0.3)
    B, L = 32, 48
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, 12, 8, seed=3)
    gen = dict(do_sample=True, top_k=50, suppress_tokens=[5], sequence_bias={(3, 7): -2.0}, exponential_decay_length_penalty=(40, 1.2),
               renormalize_logits=True)
    out = model.generate(encoder_outputs=(enc.to(DEV).bfloat16(),), attention_mask=enc_mask.to(DEV),
                         prompt_hidden_states=prompt.to(DEV).bfloat16(), prompt_attention_mask=prompt_mask.to(DEV), max_length=L,
                         return_dict_in_generate=True, output_scores=True, output_logits=True, seed=5, **gen)
    sess = next(iter(model.decoder.engine._sessions.values()))   # one session of 32 rows: its raw (un-delayed) history
    raw = sess.raw_ids[:, :out.raw_ids.shape[1]].cpu().numpy()
    parler = ParlerLogitsProcessorOracle(cfg.eos_token_id, cfg.num_codebooks, B)
    assert len(out.scores) == raw.shape[1] - 1
    for t in range(len(out.scores)):
        got = out.scores[t].cpu().numpy()
        want = lo.process_scores(out.logits[t].cpu().numpy(), raw[:, :t + 1], parler, gen, 1, L)
        kept_g, kept_w = np.isfinite(got), np.isfinite(want)
        assert (kept_g != kept_w).sum() <= 2, t
        both = kept_g & kept_w
        assert np.all(np.abs(got[both] - want[both]) <= LOG_SOFTMAX_TOL * np.maximum(1.0, np.abs(want[both]))), t
        assert (got[:, 5] == -np.inf).all()


def _margins(scores):
    fin = [np.sort(np.where(np.isfinite(s), s, -1e30), -1) for s in scores]
    return [float((f[:, -1] - f[:, -2]).min()) for f in fin]


@pytest.mark.gpu
@pytest.mark.parametrize("knobs", [
    dict(sequence_bias={(7,): 3.0, (3, 7): -2.0, (7, 7): -6.0, (12, 5): 2.5}),
    dict(suppress_tokens=[7, 12, 30], begin_suppress_tokens=[0, 1, 2, 3, 4, 5]),
    dict(forced_eos_token_id=9, sequence_bias={(20,): 1.0}, renormalize_logits=True),
], ids=["sequence_bias", "suppress", "forced_eos"])
def test_greedy_matches_oracle(knobs):
    """fp32 tiny, greedy, free-running: token for token against the oracle up to the first step whose top-2 margin is below 1e-4
    (past a near-tie, the device's logits may legitimately pick the other id)."""
    from oracle.decoder import OracleDecoder
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    w, model = _model(cfg, seed=30, head_std=0.5)
    B, S, P, L = 4, 8, 4, 40
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=3)
    gen = dict(max_length=L, do_sample=False, **knobs)
    ref = lo.generate_tokens(OracleDecoder(cfg, w, torch.float32), cfg, enc, enc_mask, prompt, prompt_mask, gen)
    m = _margins(ref["scores"])
    n = next((t for t, v in enumerate(m) if v < 1e-4), len(m))
    assert n >= 10, f"near-tie at step {n}; pick another seed"
    from parler_tts_b200.modeling import GenerationConfig, resolve_logits_ext
    sess = model.decoder.engine.session(B, P, S, P + L)
    sess.begin(L, do_sample=False, lext=resolve_logits_ext(GenerationConfig(**gen), 1, L, cfg.vocab_size, cfg.eos_token_id))
    sess.prefill(prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
    sess.sample()
    sess.decode_steps(L - 2)
    torch.cuda.synchronize()
    cur = int(sess.state[0].item())
    raw = sess.raw_ids[:, :cur].cpu().numpy()   # the raw history, as the oracle keeps it
    assert np.array_equal(raw[:, :n + 1], ref["raw_ids"][:, :n + 1])
    if n == len(m):
        assert np.array_equal(raw, ref["raw_ids"])


@pytest.mark.gpu
def test_exponential_decay_ends_utterances_near_start():
    """A large factor: every utterance ends within a few frames of the regulation start; the same call without it runs longer."""
    from tests.helpers import synth_inputs
    cfg = tiny_cfg(max_position_embeddings=256)
    _, model = _model(cfg, seed=30, head_std=0.5)
    B, L, start = 4, 120, 10
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, 8, 4, seed=3)
    kw = dict(encoder_outputs=(enc.to(DEV),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV),
              prompt_attention_mask=prompt_mask.to(DEV), do_sample=True, top_k=0, max_length=L, return_codes=True, seed=9)
    _, a = model.generate(exponential_decay_length_penalty=(start, 50.0), **kw)
    _, b = model.generate(**kw)
    K = cfg.num_codebooks
    ra = a.raw_ids.cpu().numpy()
    assert ra.shape[1] <= start + 1 + 2 * K + 2, ra.shape
    assert b.raw_ids.shape[1] > ra.shape[1] + 5, (b.raw_ids.shape, ra.shape)
    first_eos = [(np.argmax(r == cfg.eos_token_id) if (r == cfg.eos_token_id).any() else L) for r in ra]
    assert max(first_eos) <= start + 1 + 2 * K


@pytest.mark.gpu
@pytest.mark.parametrize("do_sample", [True, False], ids=["sampled", "greedy"])
def test_renormalize_keeps_tokens_and_audio(do_sample):
    """renormalize_logits: ids, codes and waveform bit-identical with and without it; the scores are log_softmax of the scores
    without it, within LOG_SOFTMAX_TOL."""
    from tests.helpers import synth_inputs
    cfg = mini_cfg(num_hidden_layers=4)
    _, model = _model(cfg, seed=21, dtype=torch.bfloat16, head_std=0.3)
    B, L = 6, 40
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, 12, 8, seed=6)
    kw = dict(encoder_outputs=(enc.to(DEV).bfloat16(),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV).bfloat16(),
              prompt_attention_mask=prompt_mask.to(DEV), do_sample=do_sample, top_k=50, max_length=L, seed=3,
              return_dict_in_generate=True, output_scores=True)
    a = model.generate(renormalize_logits=True, **kw)
    b = model.generate(**kw)
    assert torch.equal(a.raw_ids, b.raw_ids) and torch.equal(a.audio_codes, b.audio_codes)
    assert torch.equal(a.sequences, b.sequences)
    for t, (sa, sb) in enumerate(zip(a.scores, b.scores)):
        _compare(sa.cpu().numpy(), lo.log_softmax(sb.cpu().numpy()), dict(renormalize_logits=True), t)


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
    """Every stage that can change nothing here -- a bias of 0.0, suppress lists of an id already masked, InfNan on finite logits,
    a decay factor of 1, renormalize_logits -- runs every token as step kernel + EXT sampler: the ids equal the default path's bit
    for bit (B = 32 on the cluster kernel, B = 34 in shards, PTTS_STEP=legacy, a streamer)."""
    from tests.helpers import synth_inputs
    cfg = mini_cfg(num_hidden_layers=4)
    _, model = _model(cfg, seed=21, dtype=torch.bfloat16, head_std=0.3)
    L = 40
    V = cfg.vocab_size
    noop = dict(sequence_bias={(5,): 0.0, (3, 7): 0.0}, suppress_tokens=[V - 1], begin_suppress_tokens=[V - 2], remove_invalid_values=True,
                exponential_decay_length_penalty=(2, 1.0), renormalize_logits=True)
    for B, mode, streamed in [(32, None, False), (34, None, False), (32, "legacy", False), (4, None, True)]:
        monkeypatch.delenv("PTTS_STEP", raising=False)
        if mode:
            monkeypatch.setenv("PTTS_STEP", mode)
        enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, 12, 8, seed=B)
        kw = dict(encoder_outputs=(enc.to(DEV).bfloat16(),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV).bfloat16(),
                  prompt_attention_mask=prompt_mask.to(DEV), max_length=L, min_new_tokens=L, return_codes=True, seed=11,
                  _suppress_special=True, **gen)
        runs = []
        for extra in ({}, noop):
            rec = _Rec() if streamed else None
            _, out = model.generate(streamer=rec, **kw, **extra)
            runs.append((out.raw_ids.cpu(), None if rec is None else torch.cat(rec.cols, 1)))
        assert torch.equal(runs[0][0], runs[1][0]), (B, mode)
        if streamed:
            assert torch.equal(runs[0][1], runs[1][1])
    monkeypatch.delenv("PTTS_STEP", raising=False)


ROUTE_KNOBS = dict(sequence_bias={(3, 7): -2.0, (9,): 1.0}, suppress_tokens=[4], exponential_decay_length_penalty=(6, 1.3),
                   remove_invalid_values=True)


def _route_inputs(cfg, B, seed):
    from tests.helpers import synth_inputs
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, 8, 4, seed=seed)
    return enc.to(DEV).bfloat16(), enc_mask.to(DEV), prompt.to(DEV).bfloat16(), prompt_mask.to(DEV)


@pytest.mark.gpu
def test_shards_equal_separate_sessions():
    """B = 40 (shards of 32 + 8) equals the two sessions run on their own with their row_base."""
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=7, dtype=torch.bfloat16)
    B, L = 40, 30
    enc, enc_mask, prompt, prompt_mask = _route_inputs(cfg, B, 9)
    kw = dict(do_sample=True, top_k=0, max_length=L, return_codes=True, seed=4, **ROUTE_KNOBS)
    run = lambda sl, rb: model.generate(encoder_outputs=(enc[sl],), attention_mask=enc_mask[sl], prompt_hidden_states=prompt[sl],
                                        prompt_attention_mask=prompt_mask[sl], row_base=rb, **kw)[1].raw_ids.cpu()
    full = run(slice(0, B), 0)
    a, b = run(slice(0, 32), 0), run(slice(32, B), 32 * cfg.num_codebooks)
    n = full.shape[1]
    pad = lambda t: torch.nn.functional.pad(t, (0, n - t.shape[1]), value=cfg.pad_token_id)
    assert torch.equal(full, torch.cat([pad(a), pad(b)], 0))


@pytest.mark.gpu
def test_num_return_sequences_equals_expanded_batch():
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=7, dtype=torch.bfloat16)
    B, N, L = 3, 2, 30
    enc, enc_mask, prompt, prompt_mask = _route_inputs(cfg, B, 2)
    kw = dict(do_sample=True, top_k=0, max_length=L, return_codes=True, seed=8, **ROUTE_KNOBS)
    _, a = model.generate(encoder_outputs=(enc,), attention_mask=enc_mask, prompt_hidden_states=prompt,
                          prompt_attention_mask=prompt_mask, num_return_sequences=N, **kw)
    rep = lambda t: t.repeat_interleave(N, 0)
    _, b = model.generate(encoder_outputs=(rep(enc),), attention_mask=rep(enc_mask), prompt_hidden_states=rep(prompt),
                          prompt_attention_mask=rep(prompt_mask), **kw)
    assert torch.equal(a.raw_ids, b.raw_ids)


@pytest.mark.gpu
def test_continuation_suppresses_at_column_n0():
    """With decoder_input_ids (n0 > 1), begin_suppress_tokens acts on column n0 only: the ids greedy picks there without the knob
    are -inf in step 0's scores and finite in step 1's."""
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=30, head_std=0.5)
    B, L, prefix = 3, 30, 5
    enc, enc_mask, prompt, prompt_mask = _route_inputs(cfg, B, 4)
    enc, prompt = enc.float(), prompt.float()
    codes = torch.from_numpy(np.random.default_rng(3).integers(0, 40, size=(B, cfg.num_codebooks, prefix))).to(DEV)
    kw = dict(encoder_outputs=(enc,), attention_mask=enc_mask, prompt_hidden_states=prompt, prompt_attention_mask=prompt_mask,
              decoder_input_ids=codes, do_sample=False, max_length=L, return_dict_in_generate=True, output_scores=True)
    plain = model.generate(**kw)
    n0 = plain.raw_ids.shape[1] - len(plain.scores)
    assert n0 > 1
    K = cfg.num_codebooks
    # codebook 0's column n0 is drawn (the others still hold the prefix's delayed cells there)
    picked = sorted(set(plain.raw_ids[0::K, n0].tolist()))
    out = model.generate(begin_suppress_tokens=picked, **kw)
    assert (out.scores[0][:, picked] == -float("inf")).all()
    assert not np.isin(out.raw_ids[0::K, n0].cpu().numpy(), picked).any()
    s1 = out.scores[1].cpu().numpy()
    assert np.isfinite(s1[:, picked]).any()


@pytest.mark.gpu
def test_host_driven_loop_equals_device_loop():
    """A no-op caller processor moves generate() to the host-driven loop, whose torch stages give the device loop's ids and
    scores."""
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=30, head_std=0.5)
    B, L = 3, 30
    enc, enc_mask, prompt, prompt_mask = _route_inputs(cfg, B, 5)
    kw = dict(encoder_outputs=(enc.float(),), attention_mask=enc_mask, prompt_hidden_states=prompt.float(),
              prompt_attention_mask=prompt_mask, do_sample=False, max_length=L, return_dict_in_generate=True, output_scores=True,
              forced_eos_token_id=6, begin_suppress_tokens=[1, 2], **ROUTE_KNOBS)
    dev = model.generate(**kw)
    host = model.generate(logits_processor=[lambda ids, s: s], **kw)
    assert torch.equal(dev.raw_ids, host.raw_ids)
    assert len(dev.scores) == len(host.scores)
    for sd, sh in zip(dev.scores, host.scores):
        assert _same(sd.cpu().numpy(), sh.cpu().numpy())
