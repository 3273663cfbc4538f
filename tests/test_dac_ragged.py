"""Ragged DAC decode: DACModel.decode(frame_lengths=...) and generate()'s codes -> waveform step built on it.

Row b of a ragged decode with n_b = frame_lengths[b] must equal the decode of codes[b:b+1, :, :n_b] alone, bit for bit, in
samples [0, hop*n_b), be exactly 0 after them, and never read the codes at frames >= n_b.  The GPU tests check that on the
44.1 kHz codec shape at every layer's 128-row tile edge (128 frames at the first conv, 16 after x8, 2 after x64), on the wgmma
path, the generic bf16 path (PTTS_DAC_TC=0) and fp32; and that generate() gives exactly what the per-sample loop it replaces
gave.  The host tests cover the argument checks and the frame compaction.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg

DEV = "cuda"
EDGE_LENGTHS = [0, 1, 2, 15, 16, 17, 127, 128, 129]   # + T
T_EDGE = 131


# ---- host --------------------------------------------------------------------------------------------------------------------------
def _reference_gather(codes: torch.Tensor, cs: int):
    """The reference's per-row boolean gather (modeling_parler_tts.py :3631-3633): each row's valid frames, in order."""
    out = []
    for b in range(codes.shape[0]):
        ok = (codes[b] >= cs).sum(dim=0) == 0
        out.append(codes[b][:, ok])
    return out


def test_compact_valid_frames_matches_reference_gather():
    from parler_tts_b200.modeling import compact_valid_frames
    cs, K, T = 64, 4, 23
    g = torch.Generator().manual_seed(5)
    codes = torch.randint(0, cs, (6, K, T), generator=g)
    codes[0, :, 17:] = cs                      # EOS then pad: a finished row
    codes[1, 2, 5] = cs + 3                    # one invalid id mid-row, one codebook only
    codes[1, :, 9:11] = cs + 1                 # a run of invalid frames mid-row
    codes[2] = cs                              # no valid frame
    codes[3, 0, 0] = cs                        # the first frame invalid
    codes[4, K - 1, T - 1] = 10 ** 6           # the last frame invalid
    # row 5: every frame valid
    packed, n = compact_valid_frames(codes, cs)
    assert n.dtype == torch.int64 and n.tolist() == [int((codes[b] < cs).all(0).sum()) for b in range(6)]
    assert n.tolist()[2] == 0 and n.tolist()[5] == T
    for b, ref in enumerate(_reference_gather(codes, cs)):
        assert torch.equal(packed[b, :, : n[b]], ref), b


def test_compact_valid_frames_empty_time_axis():
    from parler_tts_b200.modeling import compact_valid_frames
    packed, n = compact_valid_frames(torch.zeros(3, 4, 0, dtype=torch.int64), 64)
    assert packed.shape == (3, 4, 0) and n.tolist() == [0, 0, 0]


def test_frame_lengths_validation():
    from parler_tts_b200.dac_wrapper import _frame_lengths
    B, T = 3, 10
    assert _frame_lengths([0, 10, 4], B, T).tolist() == [0, 10, 4]
    assert _frame_lengths(torch.tensor([1, 2, 3], dtype=torch.int16), B, T).dtype == torch.int32
    assert _frame_lengths(np.array([1, 2, 3]), B, T).tolist() == [1, 2, 3]
    bad = [
        [1, 2],                                          # wrong length
        torch.tensor([[1, 2, 3]]),                       # wrong shape
        torch.tensor(3),                                 # 0-d
        [1, -1, 2],                                      # negative
        [1, 11, 2],                                      # > T
        torch.tensor([1.0, 2.0, 3.0]),                   # float dtype
        [1.0, 2, 3],                                     # float value
        torch.tensor([True, False, True]),               # bool dtype
        [True, 1, 2],
    ]
    for fl in bad:
        with pytest.raises(ValueError):
            _frame_lengths(fl, B, T)


def test_decode_rejects_bad_frame_lengths_before_any_launch():
    """decode() checks frame_lengths on the host before the codec runs; the weight blob is never touched on these calls."""
    from parler_tts_b200 import DACModel
    m = DACModel.__new__(DACModel)   # no device, no library call: validation must raise before either is needed
    m.loaded = True
    m.device = torch.device("cpu")
    from tests.helpers import product_dac_config
    m.config = product_dac_config(tiny_dac_cfg())
    codes = torch.zeros(1, 2, 4, 5, dtype=torch.int64)
    for fl in ([1], [1, 6], [-1, 2], torch.tensor([1.5, 2.0]), torch.tensor([[1, 2]])):
        with pytest.raises(ValueError):
            m.decode(codes, [None, None], frame_lengths=fl)


# ---- GPU: the codec -----------------------------------------------------------------------------------------------------------------
_DAC = {}


def _dac44(dtype):
    """The 44.1 kHz codec shape (DACConfig(): 1024 -> 1536 -> 96 channels, hop 512) with synthetic weights."""
    if dtype not in _DAC:
        import bench
        from parler_tts_b200 import DACConfig, DACModel
        cfg = DACConfig()
        _DAC[dtype] = DACModel(cfg, DEV, dtype).load_state_dict(bench.synth_dac_weights(cfg, DEV))
    return _DAC[dtype]


def _codes(B, T, seed, cs=1024, K=9):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, cs, (B, K, T), generator=g).to(DEV)


def _standalone(m, codes, lengths):
    """Each row decoded alone at its own length, zero-padded to hop * T: what a ragged decode must equal."""
    B, _, T = codes.shape
    out = torch.zeros(B, 1, T * m.hop_length, dtype=m.dtype, device=DEV)
    for b, n in enumerate(lengths):
        if n > 0:
            out[b, :, : n * m.hop_length] = m.decode(codes[b:b + 1, :, :n][None], [None]).audio_values[0]
    return out


def _check_rows(m, got, codes, lengths):
    ref = _standalone(m, codes, lengths)
    for b, n in enumerate(lengths):
        e = n * m.hop_length
        assert torch.equal(got[b, :, :e], ref[b, :, :e]), (b, n)
        assert bool((got[b, :, e:] == 0).all()) and not bool(torch.signbit(got[b, :, e:]).any()), (b, n)


_PATHS = [pytest.param(torch.bfloat16, "1", id="bf16-wgmma"), pytest.param(torch.bfloat16, "0", id="bf16-generic"),
          pytest.param(torch.float32, "1", id="fp32")]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tc", _PATHS)
def test_ragged_equals_standalone_at_tile_edges(dtype, tc, monkeypatch):
    monkeypatch.setenv("PTTS_DAC_TC", tc)
    m = _dac44(dtype)
    lengths = EDGE_LENGTHS + [T_EDGE]
    codes = _codes(len(lengths), T_EDGE, seed=1)
    got = m.decode(codes[None], [None] * len(lengths), frame_lengths=lengths).audio_values
    assert got.shape == (len(lengths), 1, T_EDGE * m.hop_length) and got.dtype == dtype
    _check_rows(m, got, codes, lengths)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tc", _PATHS[:2])
def test_ragged_equals_standalone_batch32(dtype, tc, monkeypatch):
    monkeypatch.setenv("PTTS_DAC_TC", tc)
    m = _dac44(dtype)
    T = 160
    g = torch.Generator().manual_seed(7)
    lengths = torch.randint(0, T + 1, (32,), generator=g)
    lengths[0] = T
    codes = _codes(32, T, seed=2)
    got = m.decode(codes[None], [None] * 32, frame_lengths=lengths).audio_values   # a CPU int64 tensor
    _check_rows(m, got, codes, lengths.tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tc", _PATHS)
def test_ragged_never_reads_the_tail(dtype, tc, monkeypatch):
    """Frames past each row's length hold EOS / pad / absurd ids, and the workspace holds a full-length decode's activations:
    the output is the one with valid ids there."""
    monkeypatch.setenv("PTTS_DAC_TC", tc)
    m = _dac44(dtype)
    B, T = 6, 140
    lengths = [0, 3, 17, 129, 64, 140]
    codes = _codes(B, T, seed=3)
    ref = m.decode(codes[None], [None] * B, frame_lengths=lengths).audio_values.clone()
    stale = _codes(B, T, seed=4)
    for fill in (1024, 1025, 10 ** 6, -5):
        junk = codes.clone()
        for b, n in enumerate(lengths):
            junk[b, :, n:] = fill
        m.decode(stale[None], [None] * B)   # full-length decode through the same workspace first
        got = m.decode(junk[None], [None] * B, frame_lengths=torch.tensor(lengths, dtype=torch.int32, device=DEV)).audio_values
        assert torch.equal(got, ref), fill
    with pytest.raises(IndexError):   # inside a row, an out-of-range id is still an error
        bad = codes.clone()
        bad[4, 2, 63] = 1024
        m.decode(bad[None], [None] * B, frame_lengths=lengths)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tc", _PATHS)
def test_null_frame_lengths_is_the_equal_length_decode(dtype, tc, monkeypatch):
    """frame_lengths=None, all-T lengths and the original ptts_dac_decode entry point give the same bytes."""
    from parler_tts_b200 import _lib
    monkeypatch.setenv("PTTS_DAC_TC", tc)
    m = _dac44(dtype)
    B, T = 4, 133
    codes = _codes(B, T, seed=5)
    a = m.decode(codes[None], [None] * B).audio_values
    b = m.decode(codes[None], [None] * B, frame_lengths=[T] * B).audio_values
    c = torch.empty_like(a)
    _lib.check(_lib.lib().ptts_dac_decode(C.byref(m._c), _lib.ptr(m.blob), _lib.ptr(m._ws), m._ws.numel(), _lib.ptr(codes), B, T,
                                          _lib.ptr(c), _lib.stream_ptr()))
    assert torch.equal(a.view(torch.uint8), c.view(torch.uint8))
    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


# ---- GPU: generate() against the per-sample loop it replaces -----------------------------------------------------------------------
def _per_sample_loop(dac, codes, cs, dtype):
    """The parent implementation of generate()'s per-sample branch: each row's valid frames decoded alone, zero-padded."""
    outs = []
    for b in range(codes.shape[0]):
        sample = codes[None, b]
        ok = (sample >= cs).sum(dim=(0, 1)) == 0
        if int(ok.sum()) > 0:
            outs.append(dac.decode(audio_codes=sample[:, :, ok][None], audio_scales=[None]).audio_values.reshape(-1))
        else:
            outs.append(torch.zeros(1, device=DEV, dtype=dtype))
    return torch.nn.utils.rnn.pad_sequence(outs, batch_first=True, padding_value=0), [o.shape[0] for o in outs]


def _check_generate(model, audio, out, cs):
    codes = out.audio_codes
    assert bool((codes >= cs).any()), "no invalid frame: the ragged step was not reached"
    ref, ref_len = _per_sample_loop(model.audio_encoder, codes, cs, model.dtype)
    assert audio.shape == ref.shape and audio.dtype == ref.dtype
    assert torch.equal(audio, ref)
    assert out.audios_length == ref_len
    return codes


@pytest.mark.gpu
def test_codes_to_waveform_crafted_rows():
    """An empty row, invalid frames mid-row and at the ends, on the tiny fp32 codec and the 44.1 kHz bf16 wgmma codec; and a batch
    whose rows are all empty."""
    from parler_tts_b200 import DACModel
    from parler_tts_b200.modeling import codes_to_waveform
    from oracle.weights import make_dac_weights
    from tests.helpers import product_dac_config
    dcfg = tiny_dac_cfg()
    tiny = DACModel(product_dac_config(dcfg), DEV, torch.float32).load_state_dict(make_dac_weights(dcfg, seed=2))
    for dac, cs, K in ((tiny, dcfg.codebook_size, dcfg.n_codebooks), (_dac44(torch.bfloat16), 1024, 9)):
        T = 37
        codes = _codes(5, T, seed=9, cs=cs, K=K)
        codes[0, :, 30:] = cs               # finished early
        codes[1] = cs + 1                   # no valid frame
        codes[2, 3 % K, 4] = cs + 2         # invalid mid-row
        codes[2, :, 20:25] = cs
        codes[3, :, 0] = cs                 # leading invalid frame
        got, lengths = codes_to_waveform(dac, codes, cs, dac.dtype)
        ref, ref_len = _per_sample_loop(dac, codes, cs, dac.dtype)
        assert torch.equal(got, ref) and lengths == ref_len
        assert lengths[1] == 1
        empty = torch.full((3, K, T), cs, dtype=torch.int64, device=DEV)
        got, lengths = codes_to_waveform(dac, empty, cs, dac.dtype)
        ref, ref_len = _per_sample_loop(dac, empty, cs, dac.dtype)
        assert got.shape == (3, 1) and torch.equal(got, ref) and lengths == ref_len == [1, 1, 1]


def _tiny_model(dtype, seed=51):
    from oracle.weights import make_dac_weights, make_decoder_weights
    from tests.helpers import build_product_model
    cfg, dcfg = tiny_cfg(), tiny_dac_cfg()
    w = make_decoder_weights(cfg, seed=seed, head_std=0.5)
    for k in range(cfg.num_codebooks):
        w[f"decoder.lm_heads.{k}.weight"][cfg.eos_token_id] *= 3.0
    return cfg, dcfg, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,B,kw", [(torch.float32, 3, dict(do_sample=False)),
                                        (torch.float32, 6, dict(do_sample=True, seed=3, temperature=1.3)),
                                        (torch.bfloat16, 40, dict(do_sample=True, seed=4)),   # bf16: 32 + 8 rows in two shards
                                        (torch.float32, 5, dict(do_sample=True, seed=5, num_return_sequences=2))],
                         ids=["greedy", "sampled", "shards40", "takes2"])
def test_generate_matches_per_sample_loop_tiny(dtype, B, kw):
    from tests.helpers import synth_inputs
    cfg, dcfg, model = _tiny_model(dtype)
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, 8, 4, seed=8)
    enc, prompt = enc.to(DEV, dtype), prompt.to(DEV, dtype)
    audio, out = model.generate(encoder_outputs=(enc,), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt,
                                prompt_attention_mask=prompt_mask.to(DEV), max_length=30, return_codes=True, **kw)
    codes = _check_generate(model, audio, out, dcfg.codebook_size)
    assert codes.shape[0] == B * kw.get("num_return_sequences", 1)


@pytest.mark.gpu
def test_generate_matches_per_sample_loop_mini_bf16_wgmma_codec():
    """Parler-TTS-Mini layer shape in bf16 with the 44.1 kHz codec: the codes -> waveform step runs the wgmma kernels."""
    import bench
    from oracle.weights import make_decoder_weights
    from parler_tts_b200 import DACConfig, ParlerTTSConfig, ParlerTTSForConditionalGeneration
    from tests.helpers import product_decoder_config, synth_inputs
    cfg = mini_cfg(num_hidden_layers=2, max_position_embeddings=256)
    w = make_decoder_weights(cfg, seed=21, head_std=0.3)
    for k in range(cfg.num_codebooks):
        w[f"decoder.lm_heads.{k}.weight"][cfg.eos_token_id] *= 4.0
    pc = ParlerTTSConfig(vocab_size=cfg.text_vocab_size, text_encoder={}, audio_encoder=DACConfig(), decoder=product_decoder_config(cfg))
    model = ParlerTTSForConditionalGeneration(pc, device=DEV, dtype=torch.bfloat16)
    model.load_state_dict(w, dac_state_dict=bench.synth_dac_weights(pc.audio_encoder, DEV))
    B = 12
    enc, enc_mask, _, _ = synth_inputs(cfg, B, 16, 0, seed=12)
    audio, out = model.generate(encoder_outputs=(enc.to(DEV).bfloat16(),), attention_mask=enc_mask.to(DEV), do_sample=True, seed=7,
                                max_length=48, return_codes=True)
    codes = _check_generate(model, audio, out, 1024)
    n = (codes < 1024).all(dim=1).sum(dim=1)
    assert len(set(n.tolist())) > 1, n   # rows of different lengths
