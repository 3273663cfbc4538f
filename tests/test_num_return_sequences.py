"""generate(num_return_sequences=N): N takes per description, take n of description b at output row b * N + n.

Host tests pin the validation, the utterance-group expansion of continuation codes, the session plan of a sharded batch and the
workspace arithmetic of a takes session (ptts_workspace_bytes3).  GPU tests check every output against the hand-expanded batch
(`encoder_outputs` and masks repeat_interleave'd N times, same seed): bit for bit on the cluster step kernel, PTTS_STEP=legacy and
PTTS_FUSED=0, in shards, in a continuation, with both prompt modes, with the probes, the host-driven loop and the streamer, and
through ptts_score on a takes session.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg

DEV = "cuda"


# ---- host -----------------------------------------------------------------------------------------------------------------------
def test_validation():
    from parler_tts_b200.configuration import GenerationConfig
    from parler_tts_b200.modeling import ParlerTTSForConditionalGeneration, resolve_num_return_sequences
    assert resolve_num_return_sequences(GenerationConfig(do_sample=False)) == 1        # N = 1 is today's call, greedy or not
    assert resolve_num_return_sequences(GenerationConfig(do_sample=True, num_return_sequences=5)) == 5
    for bad in (0, -2, 2.0, "2", None, True):
        with pytest.raises(ValueError, match="strictly positive integer"):
            resolve_num_return_sequences(GenerationConfig(do_sample=True, num_return_sequences=bad))
    with pytest.raises(ValueError, match="Greedy methods without beam search"):
        resolve_num_return_sequences(GenerationConfig(do_sample=False, num_return_sequences=2))
    knobs = ParlerTTSForConditionalGeneration._NEUTRAL_GENERATION_KNOBS
    assert "num_return_sequences" not in knobs
    assert {"num_beam_groups", "repetition_penalty", "length_penalty", "penalty_alpha", "bad_words_ids", "force_words_ids",
            "guidance_scale"} <= set(knobs)


def test_expand_takes_repeats_utterance_groups():
    from parler_tts_b200.modeling import expand_takes, prepare_decoder_input_ids
    B, K, n, N, bos = 3, 4, 5, 3, 65
    codes = torch.arange(B * K * n).reshape(B, K, n) % 60
    for form in (codes.reshape(B * K, n), codes, codes[None]):     # [B*K, n], [B, K, n] and generate()'s audio_codes[None]
        ids = prepare_decoder_input_ids(form, B, K, 96, bos, "cpu")
        got = expand_takes(ids, B, K, N)
        assert got.shape == (B * N * K, n + 1)
        for b in range(B):
            for j in range(N):
                u = b * N + j    # take j of utterance b: utterance b's K code rows, in codebook order
                assert torch.equal(got[u * K:(u + 1) * K], ids[b * K:(b + 1) * K]), (b, j)
    assert torch.equal(expand_takes(ids, B, K, 1), ids)


@pytest.mark.parametrize("N", [1, 3, 8, 32, 40])
def test_take_shards_cover_whole_groups(N):
    from parler_tts_b200.modeling import take_shards
    limit = 32
    for B in sorted({1, 2, max(1, 32 // N), max(1, 32 // N) + 1, max(1, 33 // N) + 1, 5}):
        shards = take_shards(B, N, limit)
        rows = []
        for d0, d1, r0, r1 in shards:
            assert 0 <= d0 < d1 <= B and r1 - r0 <= max(limit, 1)
            takes = (r1 - r0) // (d1 - d0)
            assert takes * (d1 - d0) == r1 - r0
            if N <= limit:   # whole descriptions: every take of each, floor(32 / N) descriptions per session
                assert (r0, r1) == (d0 * N, d1 * N) and takes == N and d1 - d0 <= limit // N
            else:            # one description, up to 32 of its takes; the session's takes are its rows
                assert d1 - d0 == 1 and d0 * N <= r0 < r1 <= d1 * N
            rows.extend(range(r0, r1))    # r0 is the take row: row_base = row_base + r0 * K
        assert rows == list(range(B * N)), (B, N)
        if B * N <= limit:
            assert shards == [(0, B, 0, B * N)]
    assert take_shards(7, 3, None) == [(0, 7, 0, 21)]


def test_workspace_bytes3_shrinks_cross_kv_and_mask_only():
    import torch
    from parler_tts_b200 import _lib
    from parler_tts_b200.modeling import _decoder_config_c
    from tests.helpers import product_decoder_config
    lib = _lib.lib()
    align = lambda x: (x + 255) // 256 * 256
    for cfg, dt, es in ((mini_cfg(num_hidden_layers=3), torch.bfloat16, 2), (tiny_cfg(), torch.float32, 4)):
        c = _decoder_config_c(product_decoder_config(cfg), dt)
        ckv = 2 * cfg.num_cross_attention_key_value_heads * 64
        for B, P, S, Tmax, n0 in ((12, 0, 40, 100, 1), (24, 6, 17, 80, 9)):
            def ws(fn, *extra):
                n = C.c_int64()
                _lib.check(fn(C.byref(c), B, P, S, Tmax, n0, *extra, C.byref(n)))
                return n.value
            base = ws(lib.ptts_workspace_bytes2)
            assert ws(lib.ptts_workspace_bytes3, 1) == base
            for t in (2, 3, 4, 6, 12):
                if B % t:
                    continue
                d = B // t
                # enc_mask [B/t, S] int32, and L + 1 cross strides (the GEMM output and the L layers' K/V)
                saved = align(B * S * 4) - align(d * S * 4) + (cfg.num_hidden_layers + 1) * (align(B * S * ckv * es) - align(d * S * ckv * es))
                assert ws(lib.ptts_workspace_bytes3, t) == base - saved, (B, t)
            for t in (0, -1, 5, B + 1):
                with pytest.raises(ValueError, match="takes"):
                    ws(lib.ptts_workspace_bytes3, t)


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
_MODELS = {}


def _mini():
    """Parler-TTS-Mini layer shape (H 1024, 16 heads, K 9, V 1088) in bf16, 4 layers: the cluster step kernel's shape."""
    if "mini" not in _MODELS:
        from oracle.weights import make_dac_weights, make_decoder_weights
        from tests.helpers import build_product_model
        cfg = mini_cfg(num_hidden_layers=4, max_position_embeddings=256)
        w = make_decoder_weights(cfg, seed=21, head_std=0.3)
        dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
        _MODELS["mini"] = (cfg, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16))
    return _MODELS["mini"]


def _tiny(seed=61):
    from oracle.weights import make_dac_weights, make_decoder_weights
    from tests.helpers import build_product_model
    cfg, dcfg = tiny_cfg(), tiny_dac_cfg()
    w = make_decoder_weights(cfg, seed=seed, head_std=0.5)
    return cfg, w, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=torch.float32)


def _inputs(cfg, B, S, seed, dtype=torch.bfloat16, P=0):
    from tests.helpers import synth_inputs
    enc, em, prompt, pm = synth_inputs(cfg, B, S, P, seed=seed)
    cuda = lambda t: None if t is None else t.to(DEV)
    return enc.to(DEV, dtype), cuda(em), None if prompt is None else prompt.to(DEV, dtype), cuda(pm)


def _rep(t, N):
    return None if t is None else t.repeat_interleave(N, dim=0)


def _generate(model, enc, em, N, expanded, **kw):
    """generate() with N takes, or (expanded=True) over the hand-expanded batch with num_return_sequences=1."""
    if expanded:
        return model.generate(encoder_outputs=(_rep(enc, N),), attention_mask=_rep(em, N), return_dict_in_generate=True, **kw)
    return model.generate(encoder_outputs=(enc,), attention_mask=em, num_return_sequences=N, return_dict_in_generate=True, **kw)


def _same(a, b, what):
    if isinstance(a, (tuple, list)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, f"{what}[{i}]")
        return
    if isinstance(a, torch.Tensor):
        assert a.shape == b.shape and a.dtype == b.dtype, what
        assert torch.equal(torch.nan_to_num(a.float(), nan=12345.), torch.nan_to_num(b.float(), nan=12345.)), what
        return
    assert a == b, what


def _assert_same_outputs(got, want, keys=("sequences", "audio_codes", "audios_length", "raw_ids", "scores", "logits")):
    for k in keys:
        _same(got[k], want[k], k)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["cluster", "legacy", "multi"])
def test_mini_bf16_takes_equal_expanded_batch(monkeypatch, mode):
    """Mini bf16, 4 descriptions x 4 takes: sequences, codes, raw ids, scores and logits bit-identical to the expanded batch of 16
    on the cluster step kernel, step.cu (PTTS_STEP=legacy) and the multi-kernel path (PTTS_FUSED=0)."""
    cfg, model = _mini()
    monkeypatch.delenv("PTTS_STEP", raising=False)
    monkeypatch.delenv("PTTS_FUSED", raising=False)
    if mode == "legacy":
        monkeypatch.setenv("PTTS_STEP", "legacy")
    if mode == "multi":
        monkeypatch.setenv("PTTS_FUSED", "0")
    B, N, S = 4, 4, 32
    enc, em, _, _ = _inputs(cfg, B, S, seed=3)
    kw = dict(do_sample=True, top_k=50, temperature=1.2, max_length=24, seed=7, output_scores=True, output_logits=True, return_codes=True)
    got = _generate(model, enc, em, N, False, **kw)
    sess = model.decoder.engine._sessions[(B * N, 0, S)]
    assert sess.takes == N and sess.fused == {"cluster": 2, "legacy": 1, "multi": 0}[mode]
    want = _generate(model, enc, em, N, True, **kw)
    sess = model.decoder.engine._sessions[(B * N, 0, S)]
    assert sess.takes == 1 and sess.fused == {"cluster": 2, "legacy": 1, "multi": 0}[mode]
    assert got.raw_ids.shape[0] == B * N * cfg.num_codebooks and got.audio_codes.shape[0] == B * N
    assert len(got.scores) == got.raw_ids.shape[1] - 1 and got.scores[0].shape == (B * N * cfg.num_codebooks, cfg.vocab_size)
    _assert_same_outputs(got, want)
    # the takes differ from each other (they are draws, not copies)
    codes = got.audio_codes
    assert not torch.equal(codes[0], codes[1])


@pytest.mark.gpu
@pytest.mark.parametrize("B,N", [(5, 8), (1, 40)], ids=["5x8", "1x40"])
def test_mini_bf16_sharded_takes_equal_expanded_batch(B, N):
    """Above 32 rows: sessions of whole groups of takes (5 x 8: 4 + 1 descriptions; 1 x 40: 32 + 8 takes of one description, the
    second at 32 encoder rows, below the prefill GEMM's 128-row tile) equal the expanded batch's shards of 32 + 8 rows."""
    cfg, model = _mini()
    enc, em, _, _ = _inputs(cfg, B, 32, seed=4)
    kw = dict(do_sample=True, top_k=50, max_length=20, seed=11, output_scores=True)
    got = _generate(model, enc, em, N, False, **kw)
    want = _generate(model, enc, em, N, True, **kw)
    assert got.audio_codes.shape[0] == B * N
    _assert_same_outputs(got, want, keys=("sequences", "audio_codes", "raw_ids", "scores"))


@pytest.mark.gpu
def test_mini_bf16_continuation_takes():
    """decoder_input_ids with N = 3: every take starts with its own utterance's prefix frames and equals the expanded batch."""
    cfg, model = _mini()
    B, N, S, n0, K = 2, 3, 64, 5, cfg.num_codebooks
    enc, em, _, _ = _inputs(cfg, B, S, seed=5)
    prefix = torch.randint(0, cfg.codebook_size, (B, K, n0), generator=torch.Generator().manual_seed(6)).to(DEV)
    kw = dict(do_sample=True, top_k=50, max_new_tokens=16, seed=3, output_scores=True)
    got = model.generate(encoder_outputs=(enc,), attention_mask=em, decoder_input_ids=prefix, num_return_sequences=N,
                         return_dict_in_generate=True, **kw)
    want = model.generate(encoder_outputs=(_rep(enc, N),), attention_mask=_rep(em, N), decoder_input_ids=_rep(prefix, N),
                          return_dict_in_generate=True, **kw)
    _assert_same_outputs(got, want, keys=("sequences", "audio_codes", "raw_ids", "scores"))
    for b in range(B):
        for j in range(N):
            assert torch.equal(got.audio_codes[b * N + j, :, :n0], prefix[b]), (b, j)


@pytest.mark.gpu
def test_prompt_modes_takes():
    """N = 2 with a prompt_cross_attention model (the prompt joins the shared cross states) and with a P > 0 self-attention prompt
    prefix (expanded per take): both equal the expanded batch."""
    from oracle.weights import make_dac_weights, make_decoder_weights
    from parler_tts_b200 import ParlerTTSConfig, ParlerTTSForConditionalGeneration
    from tests.helpers import product_dac_config, product_decoder_config
    cfg = tiny_cfg()
    w = make_decoder_weights(cfg, seed=13, head_std=0.5)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    pc = ParlerTTSConfig(vocab_size=cfg.text_vocab_size, text_encoder={}, audio_encoder=product_dac_config(dcfg),
                         decoder=product_decoder_config(cfg), prompt_cross_attention=True)
    xmodel = ParlerTTSForConditionalGeneration(pc, device=DEV, dtype=torch.float32)
    xmodel.load_state_dict(w, dac_state_dict=make_dac_weights(dcfg, seed=2))
    B, N, S, P = 3, 2, 10, 7
    enc, em, _, _ = _inputs(cfg, B, S, seed=8, dtype=torch.float32)
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(0, cfg.text_vocab_size, (B, P), generator=g).to(DEV)
    pm = torch.ones(B, P, dtype=torch.long, device=DEV)
    pm[0, :2] = 0
    kw = dict(do_sample=True, top_k=20, max_length=24, seed=5, return_dict_in_generate=True, output_scores=True)
    got = xmodel.generate(encoder_outputs=(enc,), attention_mask=em, prompt_input_ids=ids, prompt_attention_mask=pm,
                          num_return_sequences=N, **kw)
    want = xmodel.generate(encoder_outputs=(_rep(enc, N),), attention_mask=_rep(em, N), prompt_input_ids=_rep(ids, N),
                           prompt_attention_mask=_rep(pm, N), **kw)
    _assert_same_outputs(got, want, keys=("sequences", "audio_codes", "raw_ids", "scores"))

    cfg, _, model = _tiny()
    enc, em, prompt, pm = _inputs(cfg, B, S, seed=10, dtype=torch.float32, P=P)
    got = model.generate(encoder_outputs=(enc,), attention_mask=em, prompt_hidden_states=prompt, prompt_attention_mask=pm,
                         num_return_sequences=N, **kw)
    assert model.decoder.engine._sessions[(B * N, P, S)].takes == N
    want = model.generate(encoder_outputs=(_rep(enc, N),), attention_mask=_rep(em, N), prompt_hidden_states=_rep(prompt, N),
                          prompt_attention_mask=_rep(pm, N), **kw)
    _assert_same_outputs(got, want, keys=("sequences", "audio_codes", "raw_ids", "scores"))


@pytest.mark.gpu
def test_mini_bf16_probes_takes():
    """output_attentions / output_hidden_states: the cross-attention weights of take n (read from the shared K/V), the decoder
    attentions and hidden states equal those of row b * N + n of the expanded run."""
    cfg, model = _mini()
    B, N, S = 2, 2, 64
    enc, em, _, _ = _inputs(cfg, B, S, seed=12)
    kw = dict(do_sample=True, top_k=50, max_length=12, seed=2, output_attentions=True, output_hidden_states=True)
    got = _generate(model, enc, em, N, False, **kw)
    want = _generate(model, enc, em, N, True, **kw)
    assert got.cross_attentions[1][0].shape[0] == B * N
    _assert_same_outputs(got, want, keys=("raw_ids", "cross_attentions", "decoder_attentions", "decoder_hidden_states"))


@pytest.mark.gpu
def test_host_loop_and_streamer_takes():
    """The host-driven loop (a pass-through logits_processor) sees B * N * K rows and draws what it draws over the expanded
    batch; ParlerTTSStreamer(incremental=True) yields [B * N, n] chunks that concatenate to the returned audio."""
    from parler_tts_b200 import ParlerTTSStreamer
    cfg, _, model = _tiny()
    B, N, S = 2, 2, 8
    enc, em, _, _ = _inputs(cfg, B, S, seed=14, dtype=torch.float32)
    seen = []

    def passthrough(ids, scores):
        seen.append(scores.shape[0])
        return scores
    kw = dict(do_sample=True, top_k=20, max_length=20, seed=1, logits_processor=[passthrough], output_scores=True)
    got = _generate(model, enc, em, N, False, **kw)
    assert seen and set(seen) == {B * N * cfg.num_codebooks}
    want = _generate(model, enc, em, N, True, **kw)
    _assert_same_outputs(got, want, keys=("raw_ids", "audio_codes", "scores"))

    st = ParlerTTSStreamer(model, device=DEV, play_steps=6, incremental=True)
    audio = model.generate(encoder_outputs=(enc,), attention_mask=em, num_return_sequences=N, do_sample=True, top_k=20,
                           max_length=40, seed=4, streamer=st, _suppress_special=True)
    chunks = [c for c in st]
    assert all(c.shape[0] == B * N for c in chunks) and sum(c.shape[-1] > 0 for c in chunks) >= 2
    total = np.concatenate(chunks, axis=-1)
    full = audio.float().cpu().numpy()
    assert total.shape == full.shape
    assert np.abs(total - full).max() < 1e-4


@pytest.mark.gpu
def test_mini_bf16_scoring_takes():
    """Best-of-N: the N takes scored with forward(labels=...) under their description give finite per-utterance losses, and
    ptts_score on a takes session (one cross K/V per description) gives the expanded batch's token losses bit for bit."""
    cfg, model = _mini()
    B, N, S, K = 3, 4, 64, cfg.num_codebooks
    enc, em, _, _ = _inputs(cfg, B, S, seed=15)
    out = _generate(model, enc, em, N, False, do_sample=True, top_k=50, max_length=16, seed=9)
    ids = out.raw_ids                       # [B*N*K, T+1], delayed
    T = ids.shape[1] - 1
    dec = ids[:, :T].contiguous()
    labels = ids[:, 1:].reshape(B * N, K, T).transpose(1, 2).contiguous()
    res = model(encoder_outputs=(_rep(enc, N),), attention_mask=_rep(em, N), decoder_input_ids=dec, labels=labels)
    per_take = res.token_losses.double().sum(dim=(1, 2))
    assert per_take.shape == (B * N,) and bool(torch.isfinite(per_take).all()) and bool((per_take > 0).all())
    sess = model.decoder.engine.session(B * N, 0, S, T, max_input_len=T, takes=N)
    nll = torch.empty(B * N, T, K, dtype=torch.float32, device=DEV)
    sess.score(None, None, enc, em, dec, labels, nll)
    torch.cuda.synchronize()
    assert torch.equal(nll, res.token_losses)
