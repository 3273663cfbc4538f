"""ContinuousEngine: online continuous batching, with requests submitted, cancelled and length-limited while the batch decodes.

Host tests pin submit()'s and cancel()'s checks, the rejections at creation, the left padding and the per-slot limits of
slot_outputs.  GPU tests hold the engine against generate_continuous() over the same list, bit for bit: requests arriving in
waves (one of them while the engine is idle), per-request max_new_tokens down to the delay pattern's 2K - 2, and cancellation of
a queued and of a live request.  They pass `encoder_outputs`, so no text encoder affects the bits.
"""
from types import SimpleNamespace

import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg

DEV = "cuda"


# ---- host -----------------------------------------------------------------------------------------------------------------------
def _stub_engine(K=4, L=41, S=6, P=3):
    """An engine over a stand-in model whose conditioning passes `encoder_outputs` and the prompt states through: enough for
    submit() and cancel(), which launch nothing."""
    from parler_tts_b200.modeling import ContinuousEngine

    def conditioning(caller, input_ids, attention_mask, encoder_outputs, prompt_input_ids, prompt_attention_mask, prompt_hidden, **kw):
        return encoder_outputs[0], attention_mask, prompt_hidden, prompt_attention_mask if prompt_hidden is not None else None, None, None

    model = SimpleNamespace(config=SimpleNamespace(decoder=SimpleNamespace(num_codebooks=K), audio_encoder=SimpleNamespace(codebook_size=16)),
                            audio_encoder=SimpleNamespace(config=SimpleNamespace(decoder_rates=[2, 2])), _conditioning=conditioning)
    return ContinuousEngine(model, SimpleNamespace(max_length=L), 4, 8, S, P, False, False)


def test_submit_checks():
    eng = _stub_engine(K=4, L=41, S=6, P=3)
    enc, prompt = torch.randn(1, 6, 8), torch.randn(1, 3, 8)
    with pytest.raises(ValueError, match="max_description_length = 6"):
        eng.submit(encoder_outputs=(torch.randn(1, 7, 8),), prompt_hidden_states=prompt)
    with pytest.raises(ValueError, match="max_prompt_length = 3"):
        eng.submit(encoder_outputs=(enc,), prompt_hidden_states=torch.randn(1, 4, 8))
    with pytest.raises(ValueError, match="needs a prompt"):
        eng.submit(encoder_outputs=(enc,))
    with pytest.raises(ValueError, match="one request"):
        eng.submit(encoder_outputs=(torch.randn(2, 6, 8),), prompt_hidden_states=torch.randn(2, 3, 8))
    for m in (5, 41, 0, -1):   # outside [2K - 2, bound] = [6, 40]
        with pytest.raises(ValueError, match="max_new_tokens"):
            eng.submit(encoder_outputs=(enc,), prompt_hidden_states=prompt, max_new_tokens=m)
    for m in (6.0, True, "6"):
        with pytest.raises(ValueError, match="max_new_tokens"):
            eng.submit(encoder_outputs=(enc,), prompt_hidden_states=prompt, max_new_tokens=m)
    assert eng.idle and eng.step() == [] and eng._live is None
    assert [eng.submit(encoder_outputs=(enc,), prompt_hidden_states=prompt, max_new_tokens=m) for m in (6, 23, 40, None)] == [0, 1, 2, 3]
    assert [r[4] for r in eng._reqs] == [7, 24, 41, 41] and not eng.idle
    no_prompt = _stub_engine(P=0)
    with pytest.raises(ValueError, match="max_prompt_length = 0"):
        no_prompt.submit(encoder_outputs=(enc,), prompt_hidden_states=prompt)
    assert no_prompt.submit(encoder_outputs=(enc[:, 2:],)) == 0
    short = _stub_engine(K=4, L=6)   # max_length below 2K - 1: no per-request limit at all
    with pytest.raises(ValueError, match="no per-request max_new_tokens"):
        short.submit(encoder_outputs=(enc,), prompt_hidden_states=prompt, max_new_tokens=5)
    assert short.submit(encoder_outputs=(enc,), prompt_hidden_states=prompt) == 0


def test_cancel_checks():
    eng = _stub_engine()
    enc, prompt = torch.randn(1, 6, 8), torch.randn(1, 3, 8)
    for _ in range(3):
        eng.submit(encoder_outputs=(enc,), prompt_hidden_states=prompt)
    for bad in (3, -1, 1.0, True, "0"):
        with pytest.raises(ValueError, match="no request"):
            eng.cancel(bad)
    assert eng.cancel(1) is True and eng.cancel(1) is False
    assert list(eng._queue) == [0, 2] and eng._reqs[1] is None
    assert eng.cancel(0) and eng.cancel(2) and eng.idle and eng.step() == []


def test_left_padding():
    from parler_tts_b200.modeling import left_pad
    x = torch.randn(1, 3, 4)
    got, m = left_pad(x, torch.tensor([[0, 1, 1]]), 5, "description")
    assert torch.equal(got[:, 2:], x) and torch.equal(got[:, :2], torch.zeros(1, 2, 4)) and m.tolist() == [[0, 0, 0, 1, 1]]
    got, m = left_pad(x, None, 4, "prompt")
    assert torch.equal(got[:, 1:], x) and float(got[:, 0].abs().sum()) == 0 and m.tolist() == [[0, 1, 1, 1]]
    got, m = left_pad(x, None, 3, "prompt")
    assert got is x and m is None                          # full length: kept as given
    assert left_pad(None, None, 3, "prompt") == (None, None)
    with pytest.raises(ValueError, match="max_prompt_length = 2"):
        left_pad(x, None, 2, "prompt")
    # the padding a batch of synth_inputs holds: a row's shorter description sits right-aligned behind a zero mask
    from tests.helpers import synth_inputs
    enc, em, prompt, pm = synth_inputs(tiny_cfg(), 3, 9, 5, seed=2)
    for b in range(3):
        s = int(em[b].sum())
        got, m = left_pad(enc[b:b + 1, 9 - s:], em[b:b + 1, 9 - s:], 9, "description")
        assert torch.equal(got, enc[b:b + 1]) and torch.equal(m, em[b:b + 1]), b


def test_creation_rejections():
    from parler_tts_b200.modeling import ParlerTTSForConditionalGeneration
    for kw in (dict(batch_size=0), dict(refill_every=True), dict(stream=1), dict(max_description_length=0),
               dict(max_description_length=None), dict(max_description_length=4, max_prompt_length=-1)):
        with pytest.raises(ValueError, match="batch_size|refill_every|stream|max_description_length|max_prompt_length"):
            ParlerTTSForConditionalGeneration.continuous_engine(SimpleNamespace(), **{"max_description_length": 4, **kw})
    from parler_tts_b200.configuration import GenerationConfig
    m = ParlerTTSForConditionalGeneration.__new__(ParlerTTSForConditionalGeneration)
    m.generation_config = GenerationConfig()
    for kw, name in ((dict(output_scores=True), "output_scores"), (dict(forced_eos_token_id=3), "forced_eos_token_id"),
                     (dict(streamer=object()), "streamer"), (dict(decoder_input_ids=torch.zeros(1, 2)), "decoder_input_ids"),
                     (dict(num_beams=2), "num_beams"), (dict(encoder_outputs=(torch.zeros(1, 2, 3),)), "submit"),
                     (dict(max_new_tokens=0), "max_length"), (dict(foo=1), "foo")):
        with pytest.raises(ValueError, match=name):
            m.continuous_engine(max_description_length=4, **kw)


def test_slot_outputs_per_slot_limits_equal_scalar_calls():
    """slot_outputs with a tensor of per-slot limits gives each slot what the scalar call with its own limit gives it: finish,
    frames, valid count, and its codes and compaction over that limit's width."""
    from parler_tts_b200.modeling import slot_outputs
    K, ld, cs = 3, 20, 8
    g = torch.Generator().manual_seed(3)
    B = 8
    raw = torch.randint(0, cs + 2, (B, K, ld), generator=g)
    eos_last = torch.tensor([0, 7, 4, 13, 0, 12, 0, 6], dtype=torch.int32)
    shift = torch.tensor([0, 3, 1, 0, 8, 0, 4, 2], dtype=torch.int32)
    lims = torch.tensor([12, 5, 9, 12, 16, 10, 5, 6], dtype=torch.int32)
    cur = torch.tensor(12, dtype=torch.int32)
    for live in (False, True):
        got = slot_outputs(raw, eos_last, cur, shift, lims, cs, live=live)
        assert got[2].shape == (B, K, ld)
        for b in range(B):
            L = int(lims[b])
            want = slot_outputs(raw, eos_last, cur, shift, L, cs, live=live)
            for i in (0, 1, 4):
                assert int(got[i][b]) == int(want[i][b]), (live, b, i)
            for i in (2, 3):
                assert torch.equal(got[i][b, :, :L], want[i][b]), (live, b, i)


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
_MODELS = {}


def _model(kind):
    if kind not in _MODELS:
        from oracle.weights import make_dac_weights, make_decoder_weights
        from tests.helpers import build_product_model
        if kind == "mini":
            cfg = mini_cfg(num_hidden_layers=4, max_position_embeddings=512)
            w = make_decoder_weights(cfg, seed=21, head_std=0.3)
            dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
            _MODELS[kind] = (cfg, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16))
        else:
            cfg, dcfg = tiny_cfg(), tiny_dac_cfg()
            w = make_decoder_weights(cfg, seed=71, head_std=0.5)
            _MODELS[kind] = (cfg, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=torch.float32))
    return _MODELS[kind]


def _inputs(cfg, B, S, P, seed, dtype):
    from tests.helpers import synth_inputs
    enc, em, prompt, pm = synth_inputs(cfg, B, S, P, seed=seed)
    cuda = lambda t: None if t is None else t.to(DEV)
    return enc.to(DEV, dtype), cuda(em), None if prompt is None else prompt.to(DEV, dtype), cuda(pm)


# Mini-shaped bf16 with the wgmma-safe shard shapes of test_mini_bf16_sampled_requests_equal_generate (16 x (P + 1) and 16 x S
# reach 128 rows), sampled; tiny fp32 greedy
_SETUPS = {
    "mini": dict(S=16, P=9, dtype=torch.bfloat16, batch=16, every=8,
                 kw=lambda cfg: dict(do_sample=True, top_k=50, seed=13, max_new_tokens=96, sequence_bias={(cfg.eos_token_id,): 32.0})),
    "tiny": dict(S=8, P=4, dtype=torch.float32, batch=6, every=4,
                 kw=lambda cfg: dict(do_sample=False, max_new_tokens=40, min_new_tokens=3, no_repeat_ngram_size=3,
                                     sequence_bias={(cfg.eos_token_id,): 2.0})),
}


def _reference(model, inputs, batch, every, stream, kw):
    """generate_continuous() over the whole list: {request: (codes, waveform)}."""
    enc, em, prompt, pm = inputs
    run = model.generate_continuous(encoder_outputs=(enc,), attention_mask=em, prompt_hidden_states=prompt, prompt_attention_mask=pm,
                                    batch_size=batch, refill_every=every, return_codes=True, **kw)
    return {i: (codes, wav) for i, wav, codes in run}


def _submit(engine, inputs, i, **kw):
    enc, em, prompt, pm = inputs
    return engine.submit(encoder_outputs=(enc[i:i + 1],), attention_mask=em[i:i + 1], prompt_hidden_states=prompt[i:i + 1],
                         prompt_attention_mask=pm[i:i + 1], **kw)


class _Collect:
    """The engine's events per request: (codes, waveform) once final; with stream=True the chunks concatenated."""

    def __init__(self, stream):
        self.stream, self.out, self.chunks, self.after = stream, {}, {}, {}

    def add(self, events):
        for ev in events:
            r = ev[0]
            assert r not in self.out, (r, "event after the final one")
            if self.stream:
                _, chunk, final, codes = ev
                self.chunks.setdefault(r, []).append(chunk)
                if final:
                    self.out[r] = (codes, torch.cat(self.chunks[r]))
            else:
                _, wav, codes = ev
                self.out[r] = (codes, wav)

    def drain(self, engine):
        while not engine.idle:
            self.add(engine.step())


def _assert_equal(got, ref, ids):
    assert sorted(got) == sorted(ids), (sorted(got), sorted(ids))
    for i in ids:
        assert torch.equal(got[i][0], ref[i][0]), (i, "codes")
        assert torch.equal(got[i][1], ref[i][1]), (i, "waveform")


@pytest.mark.gpu
@pytest.mark.parametrize("stream", [False, True])
def test_requests_in_waves_equal_generate_continuous(stream):
    """40 Mini requests submitted in four waves between step() calls, the third while the engine is idle: every request's codes
    and waveform (with stream=True its chunks concatenated) equal its output from generate_continuous() over the whole list."""
    cfg, model = _model("mini")
    st = _SETUPS["mini"]
    N = 40
    inputs = _inputs(cfg, N, st["S"], st["P"], seed=41, dtype=st["dtype"])
    kw = st["kw"](cfg)
    ref = _reference(model, inputs, st["batch"], st["every"], False, kw)
    engine = model.continuous_engine(batch_size=st["batch"], refill_every=st["every"], max_description_length=st["S"],
                                     max_prompt_length=st["P"], stream=stream, return_codes=True, **kw)
    got = _Collect(stream)
    waves = [range(0, 12), range(12, 24), range(24, 32), range(32, 40)]
    assert [_submit(engine, inputs, i) for i in waves[0]] == list(waves[0])
    for _ in range(3):
        got.add(engine.step())
    assert [_submit(engine, inputs, i) for i in waves[1]] == list(waves[1])    # while the first wave decodes
    got.drain(engine)
    assert engine.idle and sorted(got.out) == list(range(24))
    launches = engine._live.launches
    assert engine.step() == [] and engine._live.launches == launches          # idle: nothing launched
    assert [_submit(engine, inputs, i) for i in waves[2]] == list(waves[2])    # the idle engine takes the next wave
    got.add(engine.step())
    got.add(engine.step())
    assert [_submit(engine, inputs, i) for i in waves[3]] == list(waves[3])
    got.drain(engine)
    _assert_equal(got.out, ref, range(N))
    assert {r for _, r, _ in engine.refills} >= set(range(24, 40))         # the later waves came through refills


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["mini", "tiny"])
def test_per_request_limits_equal_generate_continuous_at_that_limit(kind):
    """Requests with max_new_tokens 2K - 2, a middle value and the bound, min_new_tokens at the bound so that every request runs
    into its limit and its delay-pattern tail: each equals its row of generate_continuous(max_new_tokens=m) over the same list."""
    cfg, model = _model(kind)
    st = _SETUPS[kind]
    K = cfg.num_codebooks
    bound = 2 * K + 20
    limits = [2 * K - 2, K + 10, bound]
    N = 3 * st["batch"] + 2
    inputs = _inputs(cfg, N, st["S"], st["P"], seed=43, dtype=st["dtype"])
    kw = {**st["kw"](cfg), "min_new_tokens": bound}
    kw.pop("max_new_tokens")
    want = {i: limits[i % 3] for i in range(N)}
    engine = model.continuous_engine(batch_size=st["batch"], refill_every=st["every"], max_description_length=st["S"],
                                     max_prompt_length=st["P"], return_codes=True, max_new_tokens=bound, **kw)
    for i in range(N):
        assert _submit(engine, inputs, i, max_new_tokens=want[i] if want[i] != bound else None) == i
    got = _Collect(False)
    got.drain(engine)
    for m in limits:
        ref = _reference(model, inputs, st["batch"], st["every"], False, {**kw, "max_new_tokens": m})
        ids = [i for i in range(N) if want[i] == m]
        _assert_equal({i: got.out[i] for i in ids}, ref, ids)
        F = m + 1 - K                                           # ran to its limit: max_length - K frames
        assert all(got.out[i][0].shape[-1] == F for i in ids), (m, [got.out[i][0].shape for i in ids])


@pytest.mark.gpu
def test_set_slots2_limit_range():
    """ptts_generate_set_slots2 takes limits in [2K - 1, max_length]: 2K - 2 and max_length + 1 are refused."""
    from parler_tts_b200.modeling import GenSession
    cfg, model = _model("tiny")
    K, B, S, P, L = cfg.num_codebooks, 4, 8, 4, 30
    enc, em, prompt, pm = _inputs(cfg, B, S, P, seed=3, dtype=torch.float32)
    sess = GenSession(model.decoder.engine, B, P, S, P + L, max_input_len=2)
    sess.begin(L, do_sample=False, codebook_size=cfg.codebook_size)
    sess.prefill(prompt, pm, enc, em)
    sess.sample()
    for bad in (2 * K - 2, L + 1):
        with pytest.raises(ValueError, match="row_max_length"):
            sess.set_slots(2, [0] * B, list(range(B)), [2 * K - 1, bad, L, L])
    sess.set_slots(2, [0] * B, list(range(B)), [2 * K - 1, L, L, 2 * K])
    sess.decode_steps(4)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_cancel_queued_and_live_requests():
    """Cancel one queued request and one live request after its first streamed chunk: neither yields anything after the cancel,
    the live one's slot is refilled at the next boundary, and every other request is bit-identical to a run without cancels."""
    cfg, model = _model("mini")
    st = _SETUPS["mini"]
    N, batch, every = 32, 8, 8
    inputs = _inputs(cfg, N, st["S"], st["P"], seed=47, dtype=st["dtype"])
    kw = {**st["kw"](cfg), "sequence_bias": {(cfg.eos_token_id,): 8.0}}
    mk = lambda: model.continuous_engine(batch_size=batch, refill_every=every, max_description_length=st["S"],
                                         max_prompt_length=st["P"], stream=True, return_codes=True, **kw)
    full = _Collect(True)
    plain = mk()
    for i in range(N):
        _submit(plain, inputs, i)
    full.drain(plain)
    assert sorted(full.out) == list(range(N))

    engine = mk()
    for i in range(N):
        _submit(engine, inputs, i)
    queued = N - 3
    assert engine.cancel(queued) is True and engine.cancel(queued) is False
    got = _Collect(True)
    victim = None
    while victim is None:
        events = engine.step()
        got.add(events)
        assert events or not engine.idle
        started = [e[0] for e in events if not e[2] and e[1].numel() > 0 and e[0] not in got.out]
        if started:
            victim = started[0]
    slot = engine._slot_req.index(victim)
    n_refills = len(engine.refills)
    assert engine.cancel(victim) is True and engine.cancel(victim) is False
    events = engine.step()
    got.add(events)
    assert victim not in [e[0] for e in events]
    assert slot in [s for s, _, _ in engine.refills[n_refills:]], (slot, engine.refills[n_refills:])
    before = {r: len(c) for r, c in got.chunks.items()}
    got.drain(engine)
    assert len(got.chunks.get(victim, [])) == before[victim] and victim not in got.out
    assert queued not in got.chunks
    done = [i for i in range(N) if i not in (victim, queued)]
    _assert_equal(got.out, full.out, done)
    assert engine.cancel(done[0]) is False
