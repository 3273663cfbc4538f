"""Streamed continuous batching: generate_continuous(stream=True) and the windowed codec call under it (ptts_dac_decode3).

Host tests pin the live frame counts of slot_outputs(live=True) over a scripted history, the window plan (stream_windows) on
exhaustive small cases and against the CPU oracle codec (a scripted stream's chunks concatenate to one decode; a radius one
frame short does not), and the argument checks.  GPU tests hold ptts_dac_decode3 against ptts_dac_decode2 of each window
gathered to frame 0, bit for bit inside the emit range and exactly 0 outside it, on the wgmma, generic bf16 and fp32 paths, also
over a workspace full of NaN patterns; and every request of a streamed run against the same request of stream=False.
"""
import ctypes as C
import itertools
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg

DEV = "cuda"


# ---- host -----------------------------------------------------------------------------------------------------------------------
def test_slot_outputs_live_frames_are_prefixes_of_the_cut():
    """A scripted history read at successive boundaries: a live row's compacted frames are a prefix of every later read (the
    finished cut included), no frame appears while col < 2K - 1, and finished rows read as slot_outputs() reads them."""
    from parler_tts_b200.modeling import slot_outputs
    K, L, ld, cs = 3, 30, 34, 8
    g = torch.Generator().manual_seed(3)
    B = 5
    raw = torch.randint(0, cs, (B, K, ld), generator=g)
    raw[1, :, 9:12] = cs + 1                  # invalid frames mid-row
    raw[3, 1, 14] = cs                        # one invalid id
    eos_col = [20, 7, 3, None, 26]            # column of the last codebook's first EOS (None: runs to max_length)
    shift = torch.tensor([0, 0, 1, 2, 0], dtype=torch.int32)
    seen = {b: [] for b in range(B)}
    for cur in range(2, L + 3):
        col = cur - shift
        eos_last = torch.tensor([e + 1 if e is not None and e < int(col[b]) else 0 for b, e in enumerate(eos_col)], dtype=torch.int32)
        cur_t = torch.tensor(cur, dtype=torch.int32)
        fin, frames, codes, packed, nv = slot_outputs(raw, eos_last, cur_t, shift, L, cs, live=True)
        ref = slot_outputs(raw, eos_last, cur_t, shift, L, cs)
        for b in range(B):
            if bool(fin[b]):
                assert bool(ref[0][b]) and int(frames[b]) == int(ref[1][b]) and int(nv[b]) == int(ref[4][b]), (cur, b)
                assert torch.equal(codes[b], ref[2][b]) and torch.equal(packed[b, :, :int(nv[b])], ref[3][b, :, :int(nv[b])]), (cur, b)
            else:
                c = int(col[b])
                assert int(frames[b]) == (c - K if c >= 2 * K - 1 else 0), (cur, b)
            seen[b].append((bool(fin[b]), packed[b, :, :int(nv[b])].clone()))
    for b in range(B):
        for i, (f, p) in enumerate(seen[b]):
            for _, later in seen[b][i + 1:]:
                assert later.shape[1] >= p.shape[1] and torch.equal(later[:, :p.shape[1]], p), b
        assert seen[b][-1][0], b                  # every row finished by the end of the script


def test_stream_windows_exhaustive_small_cases():
    from parler_tts_b200.modeling import stream_windows
    for R, n, e, fin in itertools.product(range(4), range(9), range(9), (False, True)):
        if e > n:
            continue
        (start, m, lo, hi), = stream_windows([n], [e], [fin], R)
        upto = n if fin else n - R
        if not fin and upto <= e:
            assert (start, m, lo, hi) == (0, 0, 0, 0), (R, n, e, fin)
            continue
        assert start == max(0, e - R) and start + m == n, (R, n, e, fin)        # the window ends at the valid frames
        assert start + lo == e and start + hi == upto, (R, n, e, fin)           # emits what was not played, up to its context
        assert 0 <= lo <= hi <= m, (R, n, e, fin)
    assert stream_windows([5, 9], [None, 0], [True, False], 2) == [(0, 0, 0, 0), (0, 9, 0, 7)]   # no request: nothing


def _oracle_stream(dac, codes, steps, radius, hop):
    """Drive stream_windows over `codes` [K, T] revealed `steps` frames per boundary, decoding each window alone with the CPU
    oracle; returns the concatenated chunks."""
    from parler_tts_b200.modeling import stream_windows
    T, emitted, n, out = codes.shape[1], 0, 0, []
    while True:
        n = min(T, n + steps)
        fin = n == T
        (start, m, lo, hi), = stream_windows([n], [emitted], [fin], radius)
        if m > 0:
            audio = dac.decode(codes[None, None, :, start:start + m])[0, 0]
            out.append(audio[lo * hop:hi * hop])
            emitted = start + hi
        if fin:
            return torch.cat(out)


def test_stream_windows_with_the_oracle_codec_equal_one_decode():
    from oracle.dac import OracleDAC
    from oracle.weights import make_dac_weights
    from parler_tts_b200.incremental import dac_dependency_radius
    cfg = tiny_dac_cfg()
    dac = OracleDAC(cfg, make_dac_weights(cfg, seed=4))
    hop, R = int(np.prod(cfg.upsampling_ratios)), dac_dependency_radius(cfg.upsampling_ratios)
    g = torch.Generator().manual_seed(1)
    codes = torch.randint(0, cfg.codebook_size, (cfg.n_codebooks, 57), generator=g)
    full = dac.decode(codes[None, None])[0, 0]
    for steps in (1, 3, 8, 16, 57):
        got = _oracle_stream(dac, codes, steps, R, hop)
        assert got.shape == full.shape
        # torch's conv reassociates over different windows: up to 8e-6 here.  The outermost taps weigh little, so a radius one
        # frame short errs by about 1e-4 (one step per boundary), and two frames short by about 5e-2.
        assert float((got - full).abs().max()) < 2e-5, (steps, float((got - full).abs().max()))
    short = _oracle_stream(dac, codes, 1, R - 1, hop)
    assert float((short - full).abs().max()) > 5e-5


def _fake_model():
    from parler_tts_b200.configuration import GenerationConfig
    from parler_tts_b200.modeling import ParlerTTSForConditionalGeneration as M
    return SimpleNamespace(generation_config=GenerationConfig(), _MODEL_KWARGS=M._MODEL_KWARGS,
                           _NEUTRAL_GENERATION_KNOBS=M._NEUTRAL_GENERATION_KNOBS)


@pytest.mark.parametrize("stream", [1, "yes", None, 1.0])
def test_stream_must_be_a_bool(stream):
    from parler_tts_b200.modeling import ParlerTTSForConditionalGeneration
    with pytest.raises(ValueError, match="stream"):
        ParlerTTSForConditionalGeneration.generate_continuous(_fake_model(), stream=stream)


@pytest.mark.parametrize("kw, name", [
    (dict(streamer=object()), "streamer"),
    (dict(logits_processor=[lambda i, s: s]), "logits_processor"),
    (dict(output_scores=True), "output_scores"),
    (dict(forced_eos_token_id=3), "forced_eos_token_id"),
    (dict(decoder_input_ids=torch.zeros(2, 3)), "decoder_input_ids"),
    (dict(num_return_sequences=2, do_sample=True), "num_return_sequences"),
])
def test_stream_keeps_the_continuous_rejections(kw, name):
    from parler_tts_b200.modeling import ParlerTTSForConditionalGeneration
    with pytest.raises(ValueError, match=name):
        ParlerTTSForConditionalGeneration.generate_continuous(_fake_model(), stream=True, **kw)


# ---- GPU: the windowed codec call -----------------------------------------------------------------------------------------------
_DAC = {}


def _dac(kind, dtype):
    if (kind, dtype) not in _DAC:
        from parler_tts_b200 import DACConfig, DACModel
        if kind == "44k":
            import bench
            cfg = DACConfig()
            _DAC[kind, dtype] = DACModel(cfg, DEV, dtype).load_state_dict(bench.synth_dac_weights(cfg, DEV))
        else:
            from oracle.weights import make_dac_weights
            from tests.helpers import product_dac_config
            dcfg = tiny_dac_cfg()
            _DAC[kind, dtype] = DACModel(product_dac_config(dcfg), DEV, dtype).load_state_dict(make_dac_weights(dcfg, seed=2))
    return _DAC[kind, dtype]


T_CODES, T_WIN = 80, 64
# (start, n, lo, hi).  At block 0's rate (x8) a 128-row tile holds 16 frames: emit edges on either side of 16, 32 and 48.
WINDOWS = [(0, 40, 0, 40),        # window start 0, lo = 0, hi = n
           (5, 0, 0, 0),          # n = 0
           (3, 30, 12, 12),       # lo = hi
           (7, 45, 0, 20),        # lo = 0
           (11, 33, 10, 33),      # hi = n
           (2, 25, 14, 15),       # one frame
           (16, T_WIN, 10, 54),   # n = T
           (4, 50, 15, 17), (6, 50, 16, 32), (0, 64, 17, 31), (9, 60, 31, 49), (1, 61, 47, 48)]


def _decode3(m, codes, windows):
    from parler_tts_b200 import _lib
    B, _, Tc = codes.shape
    T = max(w[1] for w in windows)
    ranges = torch.tensor(windows, dtype=torch.int32).t().contiguous().to(DEV)
    audio = torch.empty(B, 1, T * m.hop_length, dtype=m.dtype, device=DEV)
    _lib.check(_lib.lib().ptts_dac_decode3(C.byref(m._c), _lib.ptr(m.blob), _lib.ptr(m._ws), m._ws.numel(), _lib.ptr(codes), B, Tc, T,
                                           _lib.ptr(ranges[0]), _lib.ptr(ranges[1]), _lib.ptr(ranges[2]), _lib.ptr(ranges[3]),
                                           _lib.ptr(audio), _lib.stream_ptr()))
    return audio


def _expected(m, codes, windows):
    """decode2 of each window gathered to frame 0, kept inside the emit range and 0 elsewhere."""
    B, K, _ = codes.shape
    T = max(w[1] for w in windows)
    gathered = torch.zeros(B, K, T, dtype=torch.int64, device=DEV)
    for b, (s, n, _, _) in enumerate(windows):
        gathered[b, :, :n] = codes[b, :, s:s + n]
    full = m.decode(gathered[None], [None] * B, frame_lengths=[w[1] for w in windows]).audio_values
    want = torch.zeros_like(full)
    h = m.hop_length
    for b, (_, _, lo, hi) in enumerate(windows):
        want[b, :, lo * h:hi * h] = full[b, :, lo * h:hi * h]
    return want


def _codes(m, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, m.config.codebook_size, (B, m.config.num_codebooks, T), generator=g).to(DEV)


_PATHS = [pytest.param("44k", torch.bfloat16, "1", id="44k-bf16-wgmma"), pytest.param("44k", torch.bfloat16, "0", id="44k-bf16-generic"),
          pytest.param("tiny", torch.float32, "1", id="tiny-fp32")]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,dtype,tc", _PATHS)
def test_decode3_equals_decode2_of_each_window(kind, dtype, tc, monkeypatch):
    monkeypatch.setenv("PTTS_DAC_TC", tc)
    m = _dac(kind, dtype)
    codes = _codes(m, len(WINDOWS), T_CODES, seed=1)
    want = _expected(m, codes, WINDOWS)
    got = _decode3(m, codes, WINDOWS)
    assert got.shape == want.shape
    for b, w in enumerate(WINDOWS):
        assert torch.equal(got[b].view(torch.uint8), want[b].view(torch.uint8)), (b, w)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,dtype,tc", _PATHS)
def test_decode3_never_reads_stale_workspace(kind, dtype, tc, monkeypatch):
    """Skipped tiles leave the workspace as it was: filled with 0xFF bytes (NaN in bf16 and fp32) before the call, none of it
    may reach an emitted sample."""
    monkeypatch.setenv("PTTS_DAC_TC", tc)
    m = _dac(kind, dtype)
    codes = _codes(m, len(WINDOWS), T_CODES, seed=2)
    want = _expected(m, codes, WINDOWS)
    m._ws.fill_(0xFF)
    got = _decode3(m, codes, WINDOWS)
    assert torch.equal(got.view(torch.uint8), want.view(torch.uint8))


@pytest.mark.gpu
def test_decode3_rejects_bad_shapes():
    from parler_tts_b200 import _lib
    m = _dac("tiny", torch.float32)
    codes = _codes(m, 2, 8, seed=3)
    r = torch.zeros(4, 2, dtype=torch.int32, device=DEV)
    audio = torch.empty(2, 1, 9 * m.hop_length, dtype=m.dtype, device=DEV)
    with pytest.raises(ValueError, match="T_codes"):   # T > T_codes
        _lib.check(_lib.lib().ptts_dac_decode3(C.byref(m._c), _lib.ptr(m.blob), _lib.ptr(m._ws), m._ws.numel(), _lib.ptr(codes), 2, 8, 9,
                                               _lib.ptr(r[0]), _lib.ptr(r[1]), _lib.ptr(r[2]), _lib.ptr(r[3]), _lib.ptr(audio),
                                               _lib.stream_ptr()))


# ---- GPU: stream=True against stream=False ----------------------------------------------------------------------------------------
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


def _check_stream(model, inputs, batch_size, refill_every, kw):
    enc, em, prompt, pm = inputs
    common = dict(encoder_outputs=(enc,), attention_mask=em, prompt_hidden_states=prompt, prompt_attention_mask=pm, batch_size=batch_size,
                  refill_every=refill_every, return_codes=True, **kw)
    ref = {i: (wav, codes) for i, wav, codes in model.generate_continuous(**common)}
    hop = model.audio_encoder.hop_length
    chunks, finals, early = {}, {}, set()
    for i, chunk, final, codes in model.generate_continuous(stream=True, **common):
        assert i not in finals, (i, "event after the final one")
        assert chunk.dim() == 1 and chunk.dtype == model.dtype and chunk.is_cuda, i
        if final:
            finals[i] = codes
        else:
            assert codes is None and chunk.shape[0] > 0 and chunk.shape[0] % hop == 0, (i, chunk.shape)
            early.add(i)
        chunks.setdefault(i, []).append(chunk)
    assert sorted(finals) == sorted(ref) == list(range(enc.shape[0]))
    for i, (wav, codes) in ref.items():
        got = torch.cat(chunks[i])
        assert got.shape == wav.shape and torch.equal(got.view(torch.uint8), wav.view(torch.uint8)), (i, "waveform")
        assert torch.equal(finals[i], codes), (i, "codes")
    assert early, "no request yielded audio before its final event"
    return early


@pytest.mark.gpu
@pytest.mark.parametrize("refill_every", [8, 16])
def test_mini_bf16_stream_equals_stream_false(refill_every):
    """48 Mini requests through 16 slots, top-k 50, an EOS bias that spreads their lengths."""
    cfg, model = _model("mini")
    inputs = _inputs(cfg, 48, 16, 9, seed=31, dtype=torch.bfloat16)
    kw = dict(do_sample=True, top_k=50, seed=13, max_new_tokens=160, sequence_bias={(cfg.eos_token_id,): 32.0})
    _check_stream(model, inputs, 16, refill_every, kw)


@pytest.mark.gpu
def test_tiny_fp32_greedy_stream_equals_stream_false():
    """Tiny fp32 greedy, 20 requests through 6 slots; min_new_tokens makes every request outlast the codec's radius."""
    cfg, model = _model("tiny")
    inputs = _inputs(cfg, 20, 8, 4, seed=5, dtype=torch.float32)
    kw = dict(do_sample=False, max_new_tokens=64, min_new_tokens=30, no_repeat_ngram_size=3, sequence_bias={(cfg.eos_token_id,): 2.0})
    _check_stream(model, inputs, 6, 4, kw)
