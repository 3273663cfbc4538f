"""generate_continuous(): N requests through the slots of one live session, a finished request's slot refilled with the next one.

Host tests pin the boundary plan (the rebased batch column keeps its parity, every offset is >= 0, idle slots park at column 1,
refill rows are padded with the last request, every slot's cut follows generate()'s rules) and every ValueError.  GPU tests import
rows into a live session and hold them against their source session over 200 steps on the three decode paths, and compare every
request of a Mini bf16 sampled run and of a tiny fp32 greedy run against the same row of one generate() over the whole list:
codes and waveform bit for bit.
"""
from types import SimpleNamespace

import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg

DEV = "cuda"


# ---- host -----------------------------------------------------------------------------------------------------------------------
def test_rebase_keeps_parity_and_parks_idle_slots():
    from parler_tts_b200.modeling import rebase_slots
    for cur in (7, 8):
        for cols in ([2, None, 5, 9, None], [3, 3, 3], [None, None], [2, 2, None]):
            new, shift = rebase_slots(cur, cols)
            assert new % 2 == cur % 2, (cur, cols)
            assert all(sh >= 0 for sh in shift), (cur, cols)
            live = [c for c in cols if c is not None]
            assert new in (max(live, default=1), max(live, default=1) + 1)
            for c, sh in zip(cols, shift):
                assert new - sh == (1 if c is None else c)
    assert rebase_slots(9, [2, 6, None]) == (7, [5, 1, 6])   # the batch column may move down
    assert rebase_slots(9, [2, 5, None]) == (5, [3, 0, 4])
    assert rebase_slots(4, [2, 5, None]) == (6, [4, 1, 5])   # one more to keep the parity


def test_refill_rows_pad_with_the_last_request():
    from parler_tts_b200.modeling import refill_rows
    t = torch.arange(10 * 3).reshape(10, 3)
    got = refill_rows(t, 4, 3, 6)
    assert torch.equal(got[:3], t[4:7]) and all(torch.equal(got[i], t[6]) for i in range(3, 6))
    assert torch.equal(refill_rows(t, 2, 5, 5), t[2:7])
    assert refill_rows(None, 0, 1, 4) is None


def test_slot_outputs_cut_what_generate_cuts():
    """Every slot's finish, frames, codes and valid-frame compaction against the per-request rules written out: frame f of
    codebook k is column f + k + 1 (n - K frames) once the history has 2K - 1 columns, every column below that; a row that ran
    to max_length has max_length columns even when its PAD (= EOS) was recorded after."""
    from parler_tts_b200.modeling import slot_outputs
    K, L, ld, cs, eos = 3, 12, 16, 8, 9
    g = torch.Generator().manual_seed(0)
    B = 6
    raw = torch.randint(0, cs + 2, (B, K, ld), generator=g)
    eos_last = torch.tensor([0, 7, 4, 13, 0, 12], dtype=torch.int32)   # slot 3: PAD recorded at column 12 after max_length
    shift = torch.tensor([0, 3, 1, 0, 8, 0], dtype=torch.int32)
    cur = torch.tensor(12, dtype=torch.int32)
    fin, frames, codes, packed, nv = slot_outputs(raw, eos_last, cur, shift, L, cs)
    assert fin.tolist() == [True, True, True, True, False, True]
    for b in range(B):
        e = int(eos_last[b])
        n = min(e, L) if e > 0 else L
        want = raw[b, :, :n] if n < 2 * K - 1 else torch.stack([raw[b, k, k + 1:k + 1 + n - K] for k in range(K)])
        F = want.shape[1]
        assert int(frames[b]) == F and torch.equal(codes[b, :, :F], want), b
        ok = [f for f in range(F) if bool((want[:, f] < cs).all())]
        assert int(nv[b]) == len(ok) and torch.equal(packed[b, :, :len(ok)], want[:, ok]), b


@pytest.mark.parametrize("kw, name", [
    (dict(forced_eos_token_id=3), "forced_eos_token_id"),
    (dict(exponential_decay_length_penalty=(2, 1.1)), "exponential_decay_length_penalty"),
    (dict(begin_suppress_tokens=[1]), "begin_suppress_tokens"),
    (dict(output_scores=True), "output_scores"),
    (dict(output_logits=True), "output_logits"),
    (dict(output_attentions=True), "output_attentions"),
    (dict(output_hidden_states=True), "output_hidden_states"),
    (dict(return_token_timestamps=True), "return_token_timestamps"),
    (dict(num_return_sequences=2, do_sample=True), "num_return_sequences"),
    (dict(streamer=object()), "streamer"),
    (dict(logits_processor=[lambda i, s: s]), "logits_processor"),
    (dict(stopping_criteria=[lambda i, s: False]), "stopping_criteria"),
    (dict(decoder_input_ids=torch.zeros(2, 3)), "decoder_input_ids"),
    (dict(decoder_attention_mask=torch.ones(1, 3)), "decoder_attention_mask"),
    (dict(input_values=torch.zeros(1, 1, 8)), "input_values"),
])
def test_rejections(kw, name):
    from parler_tts_b200.configuration import GenerationConfig
    from parler_tts_b200.modeling import check_continuous_generate
    gc = GenerationConfig()
    streamer, lp, sc = kw.pop("streamer", None), kw.pop("logits_processor", None), kw.pop("stopping_criteria", None)
    mk = {k: kw.pop(k) for k in ("decoder_input_ids", "decoder_attention_mask", "input_values") if k in kw}
    for k, v in kw.items():
        setattr(gc, k, v)
    with pytest.raises(ValueError, match=name):
        check_continuous_generate(gc, mk, streamer, lp, sc)
    # what it supports: sampling, the warpers, min_new_tokens, the n-gram ban and the other processors
    ok = GenerationConfig()
    for k, v in dict(do_sample=True, top_k=5, top_p=0.9, min_new_tokens=3, no_repeat_ngram_size=2, sequence_bias={(3,): 1.0},
                     suppress_tokens=[2], forced_bos_token_id=4, remove_invalid_values=True, renormalize_logits=True).items():
        setattr(ok, k, v)
    check_continuous_generate(ok, {})


@pytest.mark.parametrize("kw", [dict(batch_size=0), dict(batch_size=2.0), dict(refill_every=0), dict(refill_every=True)])
def test_slot_counts_are_checked_first(kw):
    from parler_tts_b200.modeling import ParlerTTSForConditionalGeneration
    with pytest.raises(ValueError, match="batch_size|refill_every"):
        ParlerTTSForConditionalGeneration.generate_continuous(SimpleNamespace(), **kw)


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


def _set_path(monkeypatch, mode):
    monkeypatch.delenv("PTTS_STEP", raising=False)
    monkeypatch.delenv("PTTS_FUSED", raising=False)
    if mode == "legacy":
        monkeypatch.setenv("PTTS_STEP", "legacy")
    if mode == "multi":
        monkeypatch.setenv("PTTS_FUSED", "0")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["cluster", "legacy", "multi"])
def test_imported_rows_continue_as_in_their_source_session(monkeypatch, mode):
    """Rows 1 and 3 of a source session (begin + prefill + first draw, cur_len 2) imported into slots 2 and 5 of a live session at
    batch column 7 (the other parity) continue bit for bit as they do in the source session: 200 steps of logits and ids, top-k
    sampling with the same Philox keys, prompt prefix and masked descriptions.  suppress_special keeps every row drawing."""
    from parler_tts_b200.modeling import GenSession
    _set_path(monkeypatch, mode)
    cfg, model = _model("mini")
    eng, K, B, S, P, L, steps = model.decoder.engine, cfg.num_codebooks, 8, 12, 9, 260, 200
    enc, em, prompt, pm = _inputs(cfg, 2 * B, S, P, seed=11, dtype=torch.bfloat16)
    kw = dict(do_sample=True, top_k=50, seed=7, suppress_special=True, codebook_size=cfg.codebook_size)
    src = GenSession(eng, B, P, S, P + L, max_input_len=2)
    src.begin(L, row_base=0, **kw)
    src.prefill(prompt[:B], pm[:B], enc[:B], em[:B])
    src.sample()
    live = GenSession(eng, B, P, S, P + L + 20, max_input_len=2)
    live.begin(L, row_base=B * K, **kw)
    live.prefill(prompt[B:], pm[B:], enc[B:], em[B:])
    live.sample()
    live.set_slots(2, [0] * B, list(range(B, 2 * B)))
    live.decode_steps(5)
    assert live.fused == src.fused == {"cluster": 2, "legacy": 1, "multi": 0}[mode]
    live.import_rows(src, [1, 3], [2, 5])
    live.set_slots(7, [0, 0, 5, 0, 0, 5, 0, 0], [B, B + 1, 1, B + 3, B + 4, 3, B + 6, B + 7])
    rows_src = torch.cat([torch.arange(K) + K, torch.arange(K) + 3 * K]).to(DEV)
    rows_live = torch.cat([torch.arange(K) + 2 * K, torch.arange(K) + 5 * K]).to(DEV)
    for t in range(steps):
        src.decode_steps(1)
        live.decode_steps(1)
        assert torch.equal(live.logits[rows_live], src.logits[rows_src]), (mode, t)
    torch.cuda.synchronize()
    assert int(src.state[0]) == 2 + steps and int(live.state[0]) == 7 + steps
    assert torch.equal(live.raw_ids[rows_live, :2 + steps], src.raw_ids[rows_src, :2 + steps]), mode
    with pytest.raises(ValueError, match="exactly one ptts_sample"):   # the source's cache now holds more than its first column
        live.import_rows(src, [0], [0])


def _check_against_generate(model, cfg, inputs, batch_size, refill_every, gen_kw):
    enc, em, prompt, pm = inputs
    N, K = enc.shape[0], cfg.num_codebooks
    ref = model.generate(encoder_outputs=(enc,), attention_mask=em, prompt_hidden_states=prompt, prompt_attention_mask=pm,
                         return_dict_in_generate=True, **gen_kw)
    run = model.generate_continuous(encoder_outputs=(enc,), attention_mask=em, prompt_hidden_states=prompt, prompt_attention_mask=pm,
                                    batch_size=batch_size, refill_every=refill_every, return_codes=True, **gen_kw)
    seen = []
    for i, wav, codes in run:
        seen.append(i)
        F = codes.shape[-1]
        assert codes.shape[0] == K and F <= ref.audio_codes.shape[-1], i
        assert torch.equal(codes, ref.audio_codes[i, :, :F]), (i, "codes")
        n = ref.audios_length[i]
        assert wav.shape[0] == n and torch.equal(wav, ref.sequences[i, :n]), (i, "waveform")
    assert sorted(seen) == list(range(N))
    return run, seen


@pytest.mark.gpu
def test_mini_bf16_sampled_requests_equal_generate():
    """80 Mini requests of varied description and prompt lengths through 32 slots, top-k 50, an EOS bias that ends them at
    spread-out steps: slots are refilled at several batch columns, and every request's codes and waveform equal its row of one
    generate() over all 80.  Its shards of 32, 32 and 16 rows and the 32-row refills all take the wgmma prefill (16 x (P + 1) and
    16 x S reach 128 rows), the condition generate_continuous states."""
    cfg, model = _model("mini")
    N, S, P = 80, 16, 9
    inputs = _inputs(cfg, N, S, P, seed=31, dtype=torch.bfloat16)
    kw = dict(do_sample=True, top_k=50, seed=13, max_new_tokens=160, sequence_bias={(cfg.eos_token_id,): 32.0})
    run, order = _check_against_generate(model, cfg, inputs, 32, 16, kw)
    assert order != sorted(order)                              # completion order, not request order
    cols = {c for _, _, c in run.refills}
    assert len(run.refills) == N - 32 and len(cols) >= 3, run.refills
    slots = [s for s, _, _ in run.refills]
    assert len(set(slots)) < len(slots)                        # some slot took more than one refill


@pytest.mark.gpu
def test_tiny_fp32_greedy_requests_equal_generate():
    """Tiny fp32, greedy with min_new_tokens and the n-gram ban: 20 requests through 6 slots equal one generate() over all 20."""
    cfg, model = _model("tiny")
    inputs = _inputs(cfg, 20, 8, 4, seed=5, dtype=torch.float32)
    kw = dict(do_sample=False, max_new_tokens=40, min_new_tokens=3, no_repeat_ngram_size=3, sequence_bias={(cfg.eos_token_id,): 2.0})
    run, _ = _check_against_generate(model, cfg, inputs, 6, 4, kw)
    assert len(run.refills) == 14
