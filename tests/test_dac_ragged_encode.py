"""Ragged DAC encode: DACModel.encode(sample_lengths=...) and generate(input_values=[clips]) built on it.

Row b of a ragged encode with n_b = sample_lengths[b] must equal the encode of input_values[b:b+1, :, :n_b] alone, bit for bit, in
its codes and its encoder output over F_b = ceil(n_b / hop) frames; its later frames hold codebook_size (no frame) and zero
latents, and its samples past n_b are never read.  The GPU tests check that on the 44.1 kHz codec shape (hop 512; 64 -> 1024
channels) and on a tiny codec, on the wgmma path, the generic bf16 path (PTTS_DAC_TC=0) and fp32.  The edge lengths put each
layer's row end on either side of the wgmma kernel's 128-row tile: 128 rows is F = 2 frames at 64 rows per frame (after the
x2 and x4 blocks), F = 16 at 8 rows per frame (after x8) and F = 128 at the last layer; and on either side of the strided convs'
super-rows (n_b one sample past or short of a frame).  The host tests cover the argument checks and generate()'s one call.
"""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

from oracle.config import dac_cfg, tiny_cfg
from oracle.weights import make_dac_weights
from tests.dac_encode_oracle import OracleDACEncoder, make_dac_encoder_weights
from tests.golden.make_dac_encode_golden import encode_cfg, weights
from tests.test_dac_encode import product_codec_config

DEV = "cuda"
HOP = 512
# samples per row: 1, hop - 1, hop, hop + 1; F = 2/3 (64-rows-per-frame tile edge), 15/16/17 (8 rows per frame), 127/128/129
# (the last layer); a frame's last sample and one past a frame; then a full-length row of an odd count
EDGE_SAMPLES = [1, HOP - 1, HOP, HOP + 1, 2 * HOP - 3, 2 * HOP + 1, 3 * HOP, 15 * HOP - 200, 16 * HOP, 16 * HOP + 1,
                17 * HOP - 1, 127 * HOP + 5, 128 * HOP, 129 * HOP - 77]
FULL = 131 * HOP - 37


# ---- host --------------------------------------------------------------------------------------------------------------------------
def test_sample_lengths_validation():
    from parler_tts_b200.dac_wrapper import _sample_lengths
    B, n = 3, 1000
    assert _sample_lengths([1, 1000, 4], B, n).tolist() == [1, 1000, 4]
    assert _sample_lengths(torch.tensor([1, 2, 3], dtype=torch.int16), B, n).dtype == torch.int32
    assert _sample_lengths(np.array([1, 2, 3]), B, n).tolist() == [1, 2, 3]
    bad = [
        [1, 2],                                          # wrong length
        torch.tensor([[1, 2, 3]]),                       # wrong shape
        torch.tensor(3),                                 # 0-d
        [1, 0, 2],                                       # 0
        [1, -1, 2],                                      # negative
        [1, 1001, 2],                                    # > samples
        torch.tensor([1.0, 2.0, 3.0]),                   # float dtype
        [1.0, 2, 3],                                     # float value
        torch.tensor([True, False, True]),               # bool dtype
        [True, 1, 2],
    ]
    for sl in bad:
        with pytest.raises(ValueError):
            _sample_lengths(sl, B, n)


def test_encode_rejects_bad_sample_lengths_before_any_launch():
    """encode() checks sample_lengths on the host before the codec runs: no library call, no device."""
    from parler_tts_b200 import DACModel
    m = DACModel.__new__(DACModel)
    m.config = product_codec_config(encode_cfg())
    m._encode = lambda *a, **k: pytest.fail("the codec ran")
    wav = torch.zeros(2, 1, 1000)
    for sl in ([1], torch.tensor([[1, 2]]), torch.tensor([1.5, 2.0]), torch.tensor([True, True]), [0, 5], [5, 1001]):
        with pytest.raises(ValueError):
            m.encode(wav, sample_lengths=sl)


def test_encode_clips_makes_one_ragged_call():
    """_encode_clips pads the clips to the longest, passes their lengths, and cuts each row's codes at its own frames."""
    from parler_tts_b200 import ParlerTTSForConditionalGeneration
    K, cs = 4, 64
    calls = []

    def encode(x, sample_lengths=None):
        calls.append((x.clone(), list(sample_lengths)))
        B, _, n = x.shape
        codes = torch.arange(B * K * math.ceil(n / HOP)).reshape(1, B, K, -1) % cs
        for b, nb in enumerate(sample_lengths):
            codes[0, b, :, math.ceil(nb / HOP):] = cs
        return types.SimpleNamespace(audio_codes=codes)

    m = ParlerTTSForConditionalGeneration.__new__(ParlerTTSForConditionalGeneration)
    m.config = types.SimpleNamespace(decoder=types.SimpleNamespace(num_codebooks=K), audio_encoder=types.SimpleNamespace(num_codebooks=K))
    m.audio_encoder = types.SimpleNamespace(encode=encode, hop_length=HOP)
    m.device = torch.device("cpu")
    clips = [torch.ones(1, 3 * HOP + 1), torch.full((HOP,), 2.0, dtype=torch.bfloat16), torch.full((1, 7), 3.0, dtype=torch.float64)]
    ids, mask = m._encode_clips(clips, 3)
    assert len(calls) == 1
    x, lens = calls[0]
    assert lens == [3 * HOP + 1, HOP, 7] and x.shape == (3, 1, 3 * HOP + 1) and x.dtype == torch.float64
    for b, (c, n) in enumerate(zip(clips, lens)):
        assert torch.equal(x[b, 0, :n], c.reshape(-1).double()) and bool((x[b, 0, n:] == 0).all())
    assert mask.tolist() == [[1, 1, 1, 1], [1, 0, 0, 0], [1, 0, 0, 0]] and mask.dtype == torch.int64
    assert ids.shape == (3, K, 4) and bool((ids[mask[:, None, :].expand_as(ids) == 0] == 0).all()) and bool((ids < cs).all())
    with pytest.raises(ValueError):
        m._encode_clips([torch.ones(5), torch.ones(5, dtype=torch.int32)], 2)


# ---- GPU: the codec -----------------------------------------------------------------------------------------------------------------
_MODELS = {}


def _codec(shape, dtype):
    """("44k", dtype): DACConfig-shaped codec (dac_cfg()) with synthetic encoder weights; ("tiny", dtype): the golden fixture's."""
    key = (shape, dtype)
    if key not in _MODELS:
        from parler_tts_b200 import DACModel
        if shape == "44k":
            cfg = dac_cfg()
            w = make_dac_weights(cfg, seed=3)
            w.update(make_dac_encoder_weights(cfg, seed=7))
        else:
            cfg = encode_cfg()
            w = weights(cfg)
        _MODELS[key] = (cfg, w, DACModel(product_codec_config(cfg), DEV, dtype).load_state_dict(w))
    return _MODELS[key]


def _waveform(B, n, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n) / 44100.0
    return (0.3 * torch.sin(2 * math.pi * 190.0 * t) + 0.1 * torch.randn(B, n, generator=g))[:, None, :].to(DEV)


def _check_rows(m, wav, lengths, codes, lat):
    """Each row against its standalone encode: codes and latents bit for bit over its frames, codebook_size and 0 after them."""
    K, cs = m.config.num_codebooks, m.config.codebook_size
    for b, n in enumerate(lengths):
        F = math.ceil(n / HOP)
        c1, l1 = m._encode(wav[b:b + 1, 0, :n], K, return_latents=True)
        assert c1.shape[-1] == F
        assert torch.equal(codes[b, :, :F], c1[0]), (b, n)
        assert torch.equal(lat[b, :F].view(torch.uint8), l1[0].view(torch.uint8)), (b, n)
        assert bool((codes[b, :, F:] == cs).all()), (b, n)
        assert bool((lat[b, F:] == 0).all()) and not bool(torch.signbit(lat[b, F:]).any()), (b, n)


_PATHS = [pytest.param(torch.bfloat16, "1", id="bf16-wgmma"), pytest.param(torch.bfloat16, "0", id="bf16-generic"),
          pytest.param(torch.float32, "1", id="fp32")]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["44k", "tiny"])
@pytest.mark.parametrize("dtype,tc", _PATHS)
def test_ragged_encode_equals_standalone_at_edges(dtype, tc, shape, monkeypatch):
    monkeypatch.setenv("PTTS_DAC_TC", tc)
    _, _, m = _codec(shape, dtype)
    lengths = EDGE_SAMPLES + [FULL]
    wav = _waveform(len(lengths), FULL, seed=1)
    K = m.config.num_codebooks
    codes, lat = m._encode(wav[:, 0], K, return_latents=True, sample_lengths=torch.tensor(lengths))
    assert codes.shape == (len(lengths), K, math.ceil(FULL / HOP)) and lat.dtype == dtype
    _check_rows(m, wav, lengths, codes, lat)
    out = m.encode(wav, sample_lengths=lengths).audio_codes   # the public surface: the same codes
    assert out.shape == (1, len(lengths), K, math.ceil(FULL / HOP)) and torch.equal(out[0], codes)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tc", _PATHS)
def test_ragged_encode_equals_standalone_batch32(dtype, tc, monkeypatch):
    monkeypatch.setenv("PTTS_DAC_TC", tc)
    _, _, m = _codec("44k", dtype)
    n = 40 * HOP + 123
    g = torch.Generator().manual_seed(23)
    lengths = torch.randint(1, n + 1, (32,), generator=g)
    lengths[0] = n
    wav = _waveform(32, n, seed=2)
    codes, lat = m._encode(wav[:, 0], m.config.num_codebooks, return_latents=True, sample_lengths=lengths.to(DEV))
    _check_rows(m, wav, lengths.tolist(), codes, lat)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tc", _PATHS)
def test_ragged_encode_never_reads_the_tail(dtype, tc, monkeypatch):
    """Samples past each row's length hold huge values or NaN, and the workspace holds a full-length encode's activations: the
    codes and latents are those of zeros there."""
    monkeypatch.setenv("PTTS_DAC_TC", tc)
    _, _, m = _codec("44k", dtype)
    lengths = [1, 700, 17 * HOP - 1, 3 * HOP, 30 * HOP + 9]
    n = max(lengths)
    wav = _waveform(len(lengths), n, seed=3)
    for b, nb in enumerate(lengths):
        wav[b, :, nb:] = 0
    K = m.config.num_codebooks
    ref_c, ref_l = m._encode(wav[:, 0], K, return_latents=True, sample_lengths=torch.tensor(lengths))
    stale = _waveform(len(lengths), n, seed=4)
    for fill in (1e30, -3e38, float("nan")):
        junk = wav.clone()
        for b, nb in enumerate(lengths):
            junk[b, :, nb:] = fill
        m._encode(stale[:, 0], K, return_latents=True)   # a full-length encode through the same workspace first
        c, l = m._encode(junk[:, 0], K, return_latents=True, sample_lengths=torch.tensor(lengths))
        assert torch.equal(c, ref_c), fill
        assert torch.equal(l.view(torch.uint8), ref_l.view(torch.uint8)), fill


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tc", _PATHS)
def test_no_sample_lengths_is_the_equal_length_encode(dtype, tc, monkeypatch):
    """sample_lengths=None, all lengths equal to samples and the original ptts_dac_encode entry point give the same bytes."""
    from parler_tts_b200 import _lib
    monkeypatch.setenv("PTTS_DAC_TC", tc)
    _, _, m = _codec("44k", dtype)
    B, n = 3, 9 * HOP + 200
    wav = _waveform(B, n, seed=5)
    K = m.config.num_codebooks
    a_c, a_l = m._encode(wav[:, 0], K, return_latents=True)
    b_c, b_l = m._encode(wav[:, 0], K, return_latents=True, sample_lengths=torch.full((B,), n))
    audio = wav[:, 0].to(dtype).contiguous()
    c_c, c_l = torch.empty_like(a_c), torch.empty_like(a_l)
    _lib.check(_lib.lib().ptts_dac_encode(C.byref(m._c), _lib.ptr(m.blob), _lib.ptr(m.encoder_blob), _lib.ptr(m._enc_ws),
                                          m._enc_ws.numel(), _lib.ptr(audio), B, n, K, _lib.ptr(c_c), _lib.ptr(c_l), _lib.stream_ptr()))
    assert torch.equal(a_c, b_c) and torch.equal(a_c, c_c)
    assert torch.equal(a_l.view(torch.uint8), b_l.view(torch.uint8)) and torch.equal(a_l.view(torch.uint8), c_l.view(torch.uint8))
    assert torch.equal(m.encode(wav).audio_codes, m.encode(wav, sample_lengths=[n] * B).audio_codes)


@pytest.mark.gpu
def test_fp32_ragged_rows_match_the_oracle(monkeypatch):
    """Tiny codec, fp32: each ragged row's latents against the CPU restatement of its own padded clip, within the tolerance of
    test_dac_encode's fixture test; its codes equal the oracle's except at near ties."""
    monkeypatch.setenv("PTTS_DAC_TC", "1")
    cfg, w, m = _codec("tiny", torch.float32)
    lengths = [1, HOP + 1, 5 * HOP - 9, 11 * HOP]
    n = max(lengths)
    wav = _waveform(len(lengths), n, seed=6)
    K = cfg.n_codebooks
    codes, lat = m._encode(wav[:, 0], K, return_latents=True, sample_lengths=torch.tensor(lengths))
    o32, o64 = OracleDACEncoder(cfg, w), OracleDACEncoder(cfg, w, torch.float64)
    for b, nb in enumerate(lengths):
        F = math.ceil(nb / HOP)
        padded = torch.nn.functional.pad(wav[b:b + 1, :, :nb].cpu(), (0, F * HOP - nb))
        ref = o32.encoder(padded)[0].numpy().T
        got = lat[b, :F].cpu().numpy()
        assert np.abs(got - ref).max() <= 2e-4 * np.abs(ref).max(), (b, np.abs(got - ref).max())
        ref_codes, sims = o64.quantize(o64.encoder(padded.double()), K)
        margins = torch.stack([s.topk(2, dim=-1).values.diff(dim=-1).neg()[..., 0] for s in sims], dim=1)[0]
        ok = (codes[b, :, :F].cpu() == ref_codes[0]) | (margins < 1e-5)
        assert bool(ok.all()), b


# ---- GPU: generate() --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_generate_from_clips_makes_one_encode_call():
    """generate(input_values=[4 clips of 3 lengths]) calls DACModel.encode once, and continues exactly as decoder_input_ids
    holding each clip's own codes with the mask of their frame counts."""
    from parler_tts_b200 import ParlerTTSConfig, ParlerTTSForConditionalGeneration
    from oracle.weights import make_decoder_weights
    from tests.helpers import product_decoder_config, synth_inputs
    cfg, dcfg = tiny_cfg(), encode_cfg()
    pc = ParlerTTSConfig(vocab_size=cfg.text_vocab_size, text_encoder={}, audio_encoder=product_codec_config(dcfg),
                         decoder=product_decoder_config(cfg))
    model = ParlerTTSForConditionalGeneration(pc, device=DEV, dtype=torch.bfloat16)
    model.load_state_dict(make_decoder_weights(cfg, seed=13, head_std=0.5), dac_state_dict=weights(dcfg))
    K, B = cfg.num_codebooks, 4
    g = torch.Generator().manual_seed(29)
    clips = [(0.3 * torch.randn(1, n, generator=g)).to(DEV) for n in (2 * HOP + 5, 6 * HOP, 2 * HOP + 5, 1)]
    enc, em, _, _ = synth_inputs(cfg, B, 6, 0, seed=19)
    kw = dict(encoder_outputs=(enc.to(DEV),), attention_mask=em.to(DEV), max_new_tokens=10, return_dict_in_generate=True,
              do_sample=True, top_k=8, seed=5)
    dac = model.audio_encoder
    real, calls = dac.encode, []
    dac.encode = lambda *a, **k: (calls.append(1), real(*a, **k))[1]
    try:
        got = model.generate(input_values=clips, **kw)
    finally:
        del dac.encode
    assert len(calls) == 1
    own = [dac.encode(c.reshape(1, 1, -1)).audio_codes.reshape(K, -1) for c in clips]
    lens = [c.shape[-1] for c in own]
    codes = torch.zeros(B, K, max(lens), dtype=torch.long, device=DEV)
    for b, c in enumerate(own):
        codes[b, :, :lens[b]] = c
    mask = (torch.arange(max(lens))[None, :] < torch.tensor(lens)[:, None]).long().to(DEV)
    want = model.generate(decoder_input_ids=codes, decoder_attention_mask=mask, **kw)
    for k in ("raw_ids", "audio_codes", "sequences"):
        assert torch.equal(got[k], want[k]), k
    assert got.audios_length == want.audios_length
