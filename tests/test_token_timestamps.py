"""generate(return_token_timestamps=True): the alignment probe, the device median filter + DTW, and the generate() plumbing.

Host tests: the CPU oracle (tests/alignment_oracle.py) against transformers' Whisper steps (tests/golden/alignment.npz), the
alignment_heads default and validation, and token_frames.  GPU tests: ptts_align_dtw against the same fixture; the alignment
rows against the decoder_attentions / cross_attentions of output_attentions=True restricted to the transcript keys and
renormalized, per head and for the default heads; timestamps against the oracle on the recorded rows; tokens and audio
bit-identical with and without the flag, in shards, with takes, continuation, masked prompts, a streamer and the host loop.
"""
import os

import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg
from tests.alignment_oracle import token_jumps

DEV = "cuda"


def _fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "alignment.npz"))
    names = sorted({k.rsplit("_", 1)[0] for k in z.files})
    return z, names


# ---- host ----------------------------------------------------------------------------------------------------------------------
def test_oracle_reproduces_transformers_fixture(golden_dir):
    z, names = _fixture(golden_dir)
    assert len(names) >= 10
    for n in names:
        filt, jumps = token_jumps(z[f"{n}_x"])
        assert np.array_equal(filt.view(np.int32), z[f"{n}_filtered"].view(np.int32)), n
        assert np.array_equal(jumps, z[f"{n}_jumps"]), n


def test_oracle_drops_masked_tokens(golden_dir):
    z, _ = _fixture(golden_dir)
    x = z["random1_x"]
    g = np.random.default_rng(0)
    wide = np.zeros((x.shape[0], x.shape[1] + 5), np.float32)
    keep = np.ones(wide.shape[1], bool)
    keep[[0, 3, 4, 9, 17]] = False
    wide[:, keep] = x
    wide[:, ~keep] = g.random((x.shape[0], 5), dtype=np.float32) * 10   # garbage: never seen by the DTW
    _, jumps = token_jumps(wide, keep.astype(np.int64))
    assert (jumps[~keep] == -1).all() and np.array_equal(jumps[keep], z["random1_jumps"])


def test_generation_config_fields_and_default_heads():
    from parler_tts_b200 import GenerationConfig
    from parler_tts_b200.modeling import resolve_alignment_heads
    gc = GenerationConfig()
    assert gc.return_token_timestamps is False and gc.alignment_heads is None
    assert gc.update(return_token_timestamps=True, alignment_heads=[[1, 0]]) == {}
    assert resolve_alignment_heads(None, 24, 16) == [[l, h] for l in range(12, 24) for h in range(16)]
    assert resolve_alignment_heads(None, 5, 2) == [[2, 0], [2, 1], [3, 0], [3, 1], [4, 0], [4, 1]]   # ceil(5 / 2) layers
    assert resolve_alignment_heads([(0, 1), [3, 0]], 4, 2) == [[0, 1], [3, 0]]


@pytest.mark.parametrize("heads", [[], [[4, 0]], [[0, 2]], [[-1, 0]], [[0, 0], [0, 0]], [[0]], [[0, 1, 2]], [[0.0, 1]], [[True, 0]], 3],
                         ids=["empty", "layer", "head", "negative", "duplicate", "short", "long", "float", "bool", "scalar"])
def test_alignment_heads_validation(heads):
    from parler_tts_b200.modeling import resolve_alignment_heads
    with pytest.raises(ValueError):
        resolve_alignment_heads(heads, 4, 2)


def test_token_frames():
    from parler_tts_b200.modeling import token_frames
    K, cs, n0 = 3, 10, 2
    ids = torch.full((3 * K, 12), 5)
    ids[0, n0 + 4] = 11                     # utterance 0: codebook 0 ends after 4 frames
    ids[K + 2, n0 + 6 + 2] = 11             # utterance 1: codebook 2's id of frame 6 (column n0 + 6 + 2) is not a code
    ids[2 * K + 1, n0] = 11                 # utterance 2: codebook 1's column n0 is frame -1 (the delay): not counted
    f = token_frames(ids, n0, K, cs)
    assert f.dtype == torch.int32 and f.tolist() == [4, 6, 12 - n0 - K + 1]
    assert token_frames(torch.full((K, n0 + 1), 5), n0, K, cs).tolist() == [0]


# ---- GPU: the median filter and DTW --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_align_dtw_matches_fixture(golden_dir):
    """Every fixture case in one batch padded to the largest shape (padded keys masked, padded frames past n_frames) and once
    more with masked garbage columns interleaved: the filtered values bit for bit, the jump frames exactly."""
    from parler_tts_b200.modeling import align_dtw
    z, names = _fixture(golden_dir)
    xs = [z[f"{n}_x"] for n in names]
    g = np.random.default_rng(5)
    rows = []
    for x in xs:
        rows.append((x, np.ones(x.shape[1], bool)))
        keep = np.ones(x.shape[1] + 3, bool)
        keep[g.choice(keep.size, 3, replace=False)] = False
        wide = np.empty((x.shape[0], keep.size), np.float32)
        wide[:, keep] = x
        wide[:, ~keep] = 5.0
        rows.append((wide, keep))
    B, T, P = len(rows), max(r[0].shape[0] for r in rows), max(r[0].shape[1] for r in rows)
    a = np.full((B, T, P), 7.0, np.float32)
    mask = np.zeros((B, P), np.int32)
    for b, (x, keep) in enumerate(rows):
        a[b, :x.shape[0], :x.shape[1]] = x
        mask[b, :x.shape[1]] = keep
    nf = torch.tensor([r[0].shape[0] for r in rows], dtype=torch.int32)
    filt, jumps = align_dtw(torch.from_numpy(a).to(DEV), nf, torch.from_numpy(mask))
    filt, jumps = filt.cpu().numpy(), jumps.cpu().numpy()
    for b, (x, keep) in enumerate(rows):
        n = names[b // 2]
        F, Pb = x.shape
        got = filt[b, :F, :Pb][:, keep]
        assert np.array_equal(got.view(np.int32), z[f"{n}_filtered"].view(np.int32)), n
        assert np.array_equal(jumps[b, :Pb][keep], z[f"{n}_jumps"]), n
        assert (jumps[b, :Pb][~keep] == -1).all() and (jumps[b, Pb:] == -1).all()
        assert np.isnan(filt[b, F:]).all()


# ---- GPU: generate() -----------------------------------------------------------------------------------------------------------
def _model(cfg, seed, dtype, head_std=0.5):
    from oracle.weights import make_dac_weights, make_decoder_weights
    from tests.helpers import build_product_model
    w = make_decoder_weights(cfg, seed=seed, head_std=head_std)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=min(cfg.codebook_size, cfg.vocab_size - 8))
    return build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=dtype)


def _kw(inputs, dtype):
    enc, enc_mask, prompt, prompt_mask = inputs
    return dict(encoder_outputs=(enc.to(DEV).to(dtype),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV).to(dtype),
                prompt_attention_mask=prompt_mask.to(DEV))


def _renorm(w, mask):
    """Eager weights [B, q, keys] restricted to the transcript keys -> renormalized over them in fp64."""
    w = w.double()
    if mask is not None:
        w = w * (mask[:, None, :].to(w.device) != 0)
    return w / w.sum(-1, keepdim=True)


def _check(model, out, heads, n0, key0, P, mask, dtype, cross=False):
    """alignment rows against the recorded attention weights, timestamps against the oracle on those rows, and the ranges."""
    from parler_tts_b200.modeling import token_frames
    BN = out.raw_ids.shape[0] // model.config.decoder.num_codebooks
    T = out.raw_ids.shape[1] - n0
    al = out.alignment
    assert al.shape == (BN, T, P) and al.dtype == torch.float32 and out.token_timestamps.shape == (BN, P)
    assert torch.isnan(al[:, T - 1]).all()   # the last column is never a decode step's input
    att = out.cross_attentions if cross else out.decoder_attentions
    m = None if mask is None else mask.to(DEV)
    if m is not None and m.shape[0] != BN:
        m = m.repeat_interleave(BN // m.shape[0], dim=0)
    rtol = 1e-5 if dtype == torch.float32 else 2.0 ** -7
    for t in range(T - 1):
        ref = sum(_renorm(att[t + 1][l][:, h, :, key0:key0 + P], m) for l, h in heads)[:, 0] / len(heads)
        live = torch.isfinite(ref).all(-1)   # a shard that ended holds NaN in both
        got = al[:, t].double()
        assert torch.equal(torch.isfinite(got).all(-1), live), t
        assert ((got[live] - ref[live]).abs() <= rtol * ref[live] + 1e-7).all(), (t, float((got[live] - ref[live]).abs().max()))
    frames = token_frames(out.raw_ids, n0, model.config.decoder.num_codebooks, model.config.audio_encoder.codebook_size)
    hop, sr = model.audio_encoder.hop_length, model.config.audio_encoder.sampling_rate
    ts = out.token_timestamps.cpu()
    for b in range(BN):
        F = int(frames[b])
        x = al[b, :F].cpu().numpy()
        _, j = token_jumps(x, None if m is None else m[b].cpu().numpy())
        want = torch.where(torch.from_numpy(j) >= 0, torch.from_numpy(j).double() * hop / sr, float("nan")).float()
        assert torch.equal(torch.nan_to_num(ts[b], nan=-1.0), torch.nan_to_num(want, nan=-1.0)), b
        v = ts[b][torch.isfinite(ts[b])]
        assert (v[1:] >= v[:-1]).all() and (v >= 0).all() and (v <= out.audios_length[b] / sr).all()


def _same(a, b):
    assert torch.equal(a.raw_ids, b.raw_ids) and torch.equal(a.sequences, b.sequences)


TS = dict(return_dict_in_generate=True, return_token_timestamps=True, output_attentions=True)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_prefix_alignment_every_head_and_default(dtype):
    from tests.helpers import synth_inputs
    cfg = tiny_cfg(rope_embeddings=True, num_attention_heads=4, num_key_value_heads=2, hidden_size=256)
    model = _model(cfg, seed=13, dtype=dtype)
    B, S, P = 3, 8, 6
    inputs = synth_inputs(cfg, B, S, P, seed=4)
    kw = _kw(inputs, dtype)
    gen = dict(do_sample=False, max_length=20)
    base = model.generate(**kw, **gen, return_dict_in_generate=True)
    L, nh = cfg.num_hidden_layers, cfg.num_attention_heads
    for heads in [[[l, h]] for l in range(L) for h in range(nh)] + [None]:
        out = model.generate(**kw, **gen, **TS, alignment_heads=heads)
        _same(out, base)
        use = heads if heads is not None else [[l, h] for l in range(L // 2, L) for h in range(nh)]
        _check(model, out, use, 1, 0, P, inputs[3], dtype)


@pytest.mark.gpu
def test_cross_alignment_every_head():
    """prompt_cross_attention: the transcript is cross keys [S, S + P) after the description's S keys."""
    from oracle.weights import make_decoder_weights
    from tests.test_prompt_cross_attention import _cross_model
    cfg = tiny_cfg()
    model = _cross_model(cfg, make_decoder_weights(cfg, seed=13, head_std=0.5), torch.float32)
    B, S, P = 2, 7, 5
    g = torch.Generator().manual_seed(3)
    enc = torch.randn(B, S, cfg.hidden_size, generator=g).to(DEV)
    em = torch.ones(B, S, dtype=torch.long, device=DEV)
    em[1, :2] = 0
    ids = torch.randint(0, 50, (B, P), generator=g).to(DEV)
    pm = torch.ones(B, P, dtype=torch.long)
    pm[0, :2] = 0
    kw = dict(encoder_outputs=(enc,), attention_mask=em, prompt_input_ids=ids, prompt_attention_mask=pm.to(DEV), do_sample=False,
              max_length=18)
    base = model.generate(**kw, return_dict_in_generate=True)
    for heads in [[[l, h]] for l in range(cfg.num_hidden_layers) for h in range(cfg.num_attention_heads)]:
        out = model.generate(**kw, **TS, alignment_heads=heads)
        _same(out, base)
        _check(model, out, heads, 1, S, P, pm, torch.float32, cross=True)
    with pytest.raises(ValueError):   # no transcript, nothing to align
        model.generate(encoder_outputs=(enc,), attention_mask=em, max_length=8, **TS)


@pytest.mark.gpu
def test_mini_bf16_batch32_bit_identical_and_matches_attentions():
    cfg = mini_cfg(num_hidden_layers=4)
    model = _model(cfg, seed=21, dtype=torch.bfloat16, head_std=0.3)
    from tests.helpers import synth_inputs
    B, S, P = 32, 12, 32
    inputs = synth_inputs(cfg, B, S, P, seed=9)
    kw = _kw(inputs, torch.bfloat16)
    gen = dict(do_sample=True, temperature=0.9, top_k=50, max_length=40, seed=3, return_dict_in_generate=True)
    base = model.generate(**kw, **gen)
    sess = next(iter(model.decoder.engine._sessions.values()))
    fused, launches0 = sess.fused, sess.launches
    ts = model.generate(**kw, **gen, return_token_timestamps=True)
    _same(ts, base)
    assert "decoder_attentions" not in ts and sess.fused == fused
    out = model.generate(**kw, **gen, return_token_timestamps=True, output_attentions=True)
    _same(out, base)
    assert torch.equal(torch.nan_to_num(out.alignment, nan=-1.0), torch.nan_to_num(ts.alignment, nan=-1.0))
    L, nh = cfg.num_hidden_layers, cfg.num_attention_heads
    _check(model, out, [[l, h] for l in range(L // 2, L) for h in range(nh)], 1, 0, P, inputs[3], torch.bfloat16)
    l1 = sess.launches
    again = model.generate(**kw, **gen)   # the flag off again: the same path and launches as the first call
    _same(again, base)
    assert sess.launches - l1 == launches0 and "alignment" not in again


@pytest.mark.gpu
def test_shards_takes_continuation_streamer_and_host_loop():
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    model = _model(cfg, seed=8, dtype=torch.bfloat16)
    B, S, P, K = 40, 8, 4, cfg.num_codebooks
    inputs = synth_inputs(cfg, B, S, P, seed=2)
    kw = _kw(inputs, torch.bfloat16)
    heads = [[1, 0], [0, 1]]
    gen = dict(do_sample=True, top_k=30, max_length=30, seed=11, return_dict_in_generate=True, alignment_heads=heads)
    base = model.generate(**kw, **gen)
    out = model.generate(**kw, **gen, return_token_timestamps=True, output_attentions=True)   # two shards of 32 and 8
    _same(out, base)
    _check(model, out, heads, 1, 0, P, inputs[3], torch.bfloat16)

    sub = {k: (v[:12] if isinstance(v, torch.Tensor) else (v[0][:12],)) for k, v in kw.items()}
    base = model.generate(**sub, **gen, num_return_sequences=3)    # 36 takes: shards of whole groups of takes
    out = model.generate(**sub, **gen, num_return_sequences=3, return_token_timestamps=True, output_attentions=True)
    _same(out, base)
    _check(model, out, heads, 1, 0, P, inputs[3][:12], torch.bfloat16)

    g = np.random.default_rng(3)
    ids = np.concatenate([np.full((12 * K, 1), cfg.bos_token_id), g.integers(0, 40, size=(12 * K, 5))], axis=1).astype(np.int64)
    cont = dict(sub, decoder_input_ids=torch.from_numpy(ids).to(DEV))
    base = model.generate(**cont, **gen)
    out = model.generate(**cont, **gen, return_token_timestamps=True, output_attentions=True)
    _same(out, base)
    _check(model, out, heads, 6, 0, P, inputs[3][:12], torch.bfloat16)

    class Cols:
        def __init__(self):
            self.cols = []

        def put(self, v):
            self.cols.append(v.clone())

        def end(self):
            pass
    small = {k: (v[:4] if isinstance(v, torch.Tensor) else (v[0][:4],)) for k, v in kw.items()}
    s0, s1 = Cols(), Cols()
    a = model.generate(**small, **gen, streamer=s0)
    b = model.generate(**small, **gen, streamer=s1, return_token_timestamps=True, output_attentions=True)
    _same(a, b)
    assert len(s0.cols) == len(s1.cols) and all(torch.equal(x, y) for x, y in zip(s0.cols, s1.cols))
    _check(model, b, heads, 1, 0, P, inputs[3][:4], torch.bfloat16)
    proc = [lambda ids, scores: scores]
    c = model.generate(**small, **gen, logits_processor=proc)
    d = model.generate(**small, **gen, logits_processor=proc, return_token_timestamps=True, output_attentions=True)
    _same(c, d)
    _check(model, d, heads, 1, 0, P, inputs[3][:4], torch.bfloat16)


@pytest.mark.gpu
def test_flag_needs_dict_return_and_valid_heads():
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    model = _model(cfg, seed=8, dtype=torch.float32)
    kw = _kw(synth_inputs(cfg, 2, 8, 4, seed=2), torch.float32)
    with pytest.raises(ValueError, match="return_dict_in_generate"):
        model.generate(**kw, max_length=8, return_token_timestamps=True)
    for heads in ([], [[2, 0]], [[0, 0], [0, 0]]):
        with pytest.raises(ValueError, match="alignment_heads"):
            model.generate(**kw, max_length=8, return_dict_in_generate=True, return_token_timestamps=True, alignment_heads=heads)
