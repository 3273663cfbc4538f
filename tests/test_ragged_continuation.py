"""generate(decoder_input_ids, decoder_attention_mask): one batch continuing from code prefixes of different lengths.

Row b of a ragged call keeps its own column and cache position (the batch's less its offset s_b = n0 - n0_b), so it computes
what generate() computes for the row alone (its own prefix, the same conditioning and seed, row_base = b * K), bit for bit.
Host tests pin the mask validation, the BOS column, the offsets, their expansion per take and slicing per shard, and what the
ragged mode refuses.  GPU tests compare the tiny model's rows against their alone runs (fp32 and bf16, greedy and sampled with
the device processors), the Mini-shape decode paths against each other and their rows against a same-size batch of the row's
own prefix (the bf16 prefill GEMM is picked by the batch's row count), the all-ones mask against no mask, takes and shards
against the hand-expanded batch, and a list of clips against the codes of each clip.
"""
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg

DEV = "cuda"


# ---- host -----------------------------------------------------------------------------------------------------------------------
def _prep(ids, mask, B=3, K=2, V=96, bos=65):
    from parler_tts_b200.modeling import prepare_ragged_decoder_input_ids
    return prepare_ragged_decoder_input_ids(ids, mask, B, K, V, bos, "cpu")


def test_mask_validation():
    ids = torch.zeros(3 * 2, 4, dtype=torch.long)
    _prep(ids, torch.tensor([[1, 1, 1, 1], [1, 1, 0, 0], [0, 0, 0, 0]]))   # an all-zero row is allowed
    with pytest.raises(ValueError, match=r"\[3, 4\]"):                       # wrong shape
        _prep(ids, torch.ones(3, 5, dtype=torch.long))
    with pytest.raises(ValueError, match=r"\[3, 4\]"):
        _prep(ids, torch.ones(3 * 4, dtype=torch.long))
    with pytest.raises(ValueError, match="right padding"):                   # a hole, left padding, a value other than 0 / 1
        _prep(ids, torch.tensor([[1, 0, 1, 0], [1, 1, 1, 1], [1, 1, 1, 1]]))
    with pytest.raises(ValueError, match="right padding"):
        _prep(ids, torch.tensor([[0, 0, 1, 1], [1, 1, 1, 1], [1, 1, 1, 1]]))
    with pytest.raises(ValueError, match="right padding"):
        _prep(ids, torch.tensor([[2, 1, 1, 1], [1, 1, 1, 1], [1, 1, 1, 1]]))
    with pytest.raises(ValueError, match="0 / 1"):
        _prep(ids, torch.ones(3, 4))


def test_padding_ids_are_not_checked_but_valid_ones_are():
    ids = torch.full((3 * 2, 4), -5, dtype=torch.long)
    ids[:, :2] = 7
    _prep(ids, torch.tensor([[1, 1, 0, 0], [1, 0, 0, 0], [0, 0, 0, 0]]))
    ids[0, 1] = 97
    with pytest.raises(ValueError, match="vocab_size"):
        _prep(ids, torch.tensor([[1, 1, 0, 0], [1, 0, 0, 0], [0, 0, 0, 0]]))


def test_bos_and_mask_prepending_and_offsets():
    from parler_tts_b200.modeling import ragged_offsets
    B, K, bos = 3, 2, 65
    ids = torch.arange(B * K * 4).reshape(B * K, 4) % 60
    mask = torch.tensor([[1, 1, 1, 0], [1, 0, 0, 0], [0, 0, 0, 0]])
    got, lens = _prep(ids, mask)
    # BOS prepended (no row starts with it): a one goes in front of the mask, n0 = 1 + the longest prefix
    assert got.shape == (B * K, 4) and bool((got[:, 0] == bos).all())
    assert torch.equal(got[:, 1:], ids[:, :3])
    assert lens.dtype == torch.int32 and lens.tolist() == [4, 2, 1]
    assert ragged_offsets(lens).tolist() == [0, 2, 3]
    # every row with frames already starts with BOS: nothing is prepended, and the trailing all-padding column is dropped
    ids2 = ids.clone()
    ids2[:, 0] = bos
    got2, lens2 = _prep(ids2, torch.tensor([[1, 1, 0, 0], [1, 1, 1, 0], [1, 0, 0, 0]]))
    assert got2.shape == (B * K, 3) and torch.equal(got2, ids2[:, :3]) and lens2.tolist() == [2, 3, 1]
    # ... and then a row without frames has no column at all
    with pytest.raises(ValueError, match="BOS"):
        _prep(ids2, torch.tensor([[1, 1, 0, 0], [1, 1, 1, 0], [0, 0, 0, 0]]))
    # the padding of a row never decides the BOS column: row 1's padding holds BOS, the valid rows do not start with it
    ids3 = ids.clone()
    ids3[2:4, :] = bos
    got3, lens3 = _prep(ids3, torch.tensor([[1, 1, 0, 0], [0, 0, 0, 0], [1, 0, 0, 0]]))
    assert bool((got3[:, 0] == bos).all()) and lens3.tolist() == [3, 1, 2]


def test_offsets_expand_per_take_and_slice_per_shard():
    """The offsets of description b repeat for each of its takes (row b * N + j), and each shard takes its rows' slice."""
    from parler_tts_b200.modeling import ragged_offsets, take_shards
    lens = torch.tensor([5, 1, 3, 2, 4], dtype=torch.int32)
    N = 8
    rows = lens.repeat_interleave(N)
    assert rows.tolist() == sum(([v] * N for v in lens.tolist()), [])
    shards = take_shards(5, N, 32)
    assert torch.equal(torch.cat([rows[r0:r1] for _, _, r0, r1 in shards]), rows)
    for d0, d1, r0, r1 in shards:
        assert rows[r0:r1].tolist() == lens[d0:d1].repeat_interleave(N).tolist()
    # a row's offset is relative to the longest input of the whole call, not of its shard
    assert ragged_offsets(rows)[r0:r1].tolist() == (5 - lens[d0:d1]).repeat_interleave(N).tolist()


def test_shard_batch_slices_the_mask_and_a_clip_list():
    from parler_tts_b200.dist import shard_batch
    B, K = 5, 2
    enc = torch.arange(B)[:, None].expand(B, 3)
    mask = torch.arange(B)[:, None].expand(B, 6)
    clips = [torch.zeros(10 + i) for i in range(B)]
    parts = [shard_batch({"encoder_outputs": enc, "decoder_attention_mask": mask, "input_values": clips}, r, 2) for r in range(2)]
    assert torch.equal(torch.cat([p["decoder_attention_mask"] for p in parts]), mask)
    assert [len(p["input_values"]) for p in parts] == [3, 2] and parts[1]["input_values"][0].shape[0] == 13


@pytest.mark.parametrize("kw,name", [
    (dict(streamer=object()), "streamer"),
    (dict(logits_processor=[lambda i, s: s]), "logits_processor"),
    (dict(stopping_criteria=[lambda i, s: False]), "stopping_criteria"),
    (dict(output_attentions=True), "output_attentions"),
    (dict(output_hidden_states=True), "output_hidden_states"),
    (dict(return_token_timestamps=True), "return_token_timestamps"),
    (dict(min_length=10), "min_length"),
])
def test_ragged_mode_rejects(kw, name):
    from parler_tts_b200.configuration import GenerationConfig
    from parler_tts_b200.modeling import check_ragged_generate
    gc = GenerationConfig()
    streamer, lp, sc = kw.pop("streamer", None), kw.pop("logits_processor", None), kw.pop("stopping_criteria", None)
    for k, v in kw.items():
        setattr(gc, k, v)
    with pytest.raises(ValueError, match=name):
        check_ragged_generate(streamer, lp, sc, gc)
    check_ragged_generate(None, None, None, GenerationConfig())   # nothing of it: accepted


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
_MODELS = {}


def _tiny(dtype):
    key = ("tiny", dtype)
    if key not in _MODELS:
        from oracle.weights import make_dac_weights, make_decoder_weights
        from tests.helpers import build_product_model
        cfg, dcfg = tiny_cfg(), tiny_dac_cfg()
        w = make_decoder_weights(cfg, seed=71, head_std=0.5)
        _MODELS[key] = (cfg, w, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=dtype))
    return _MODELS[key]


def _mini(**kw):
    key = ("mini",) + tuple(sorted(kw.items()))
    if key not in _MODELS:
        from oracle.weights import make_dac_weights, make_decoder_weights
        from tests.helpers import build_product_model
        cfg = mini_cfg(num_hidden_layers=4, max_position_embeddings=512, **kw)
        w = make_decoder_weights(cfg, seed=21, head_std=0.3)
        dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
        _MODELS[key] = (cfg, w, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16))
    return _MODELS[key]


def _inputs(cfg, B, S, P, seed, dtype):
    from tests.helpers import synth_inputs
    enc, em, prompt, pm = synth_inputs(cfg, B, S, P, seed=seed)
    cuda = lambda t: None if t is None else t.to(DEV)
    return enc.to(DEV, dtype), cuda(em), None if prompt is None else prompt.to(DEV, dtype), cuda(pm)


def _ragged_codes(cfg, lens, seed):
    """[B, K, max(lens)] random codes, padding filled with ids outside the vocabulary (never read), and the mask [B, N]."""
    B, K, N = len(lens), cfg.num_codebooks, max(max(lens), 1)
    codes = torch.randint(0, cfg.codebook_size, (B, K, N), generator=torch.Generator().manual_seed(seed))
    mask = (torch.arange(N)[None, :] < torch.tensor(lens)[:, None]).long()
    codes = torch.where(mask[:, None, :].bool(), codes, torch.full_like(codes, 10 ** 6))
    return codes.to(DEV), mask.to(DEV)


def _generate(model, enc, em, prompt, pm, **kw):
    return model.generate(encoder_outputs=(enc,), attention_mask=em, prompt_hidden_states=prompt, prompt_attention_mask=pm,
                          return_dict_in_generate=True, **kw)


def _alone(model, enc, em, prompt, pm, codes, lens, b, **kw):
    """Row b run alone: its own unpadded prefix (none for an empty one), its own conditioning, row_base = b * K."""
    K = codes.shape[1]
    cut = lambda t: None if t is None else t[b:b + 1]
    dii = None if lens[b] == 0 else codes[b:b + 1, :, :lens[b]]
    return _generate(model, cut(enc), cut(em), cut(prompt), cut(pm), decoder_input_ids=dii, row_base=b * K, **kw)


def _assert_row_equals_alone(got, alone, b, K, what=""):
    T = alone.raw_ids.shape[1]
    assert got.raw_ids.shape[1] >= T, (what, b)
    assert torch.equal(got.raw_ids[b * K:(b + 1) * K, :T], alone.raw_ids), (what, b, "raw_ids")
    F = alone.audio_codes.shape[-1]
    assert torch.equal(got.audio_codes[b, :, :F], alone.audio_codes[0]), (what, b, "audio_codes")
    n = alone.audios_length[0]
    assert got.audios_length[b] == n, (what, b, "audios_length")
    assert torch.equal(got.sequences[b, :n], alone.sequences[0, :n]), (what, b, "sequences")


def _assert_steps_equal(got, ref, b, K, what=""):
    """Per-step scores and logits of row b: entry t of the ragged call equals entry t of the run of row b alone, `ref`, while it
    ran (NaN where both are: the decay penalty of an EOS score already at -inf)."""
    same = lambda x, y: torch.equal(torch.nan_to_num(x, nan=12345.), torch.nan_to_num(y, nan=12345.))
    for t, s in enumerate(ref.scores[:len(got.scores)]):
        assert same(got.scores[t][b * K:(b + 1) * K], s), (what, b, "scores", t)
        assert torch.equal(got.logits[t][b * K:(b + 1) * K], ref.logits[t]), (what, b, "logits", t)


_SAMPLED = dict(do_sample=True, top_k=20, seed=5, min_new_tokens=4, no_repeat_ngram_size=3, sequence_bias={(3,): 1.5, (5, 7): -2.0},
                exponential_decay_length_penalty=(3, 1.2), begin_suppress_tokens=[1, 2], forced_eos_token_id=64)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["greedy", "sampled", "forced_bos"])
def test_tiny_row_equals_alone(dtype, mode):
    """B = 6, prefixes of 0, 1, 3, 9 (the batch maximum), 5 and 0 frames: every row's ids, codes, waveform, length and (sampled)
    per-step scores and logits equal generate() on that row alone.  forced_bos: a forced BOS moves begin-suppress one column
    later for the rows that continue from the BOS column alone, as it does for such a row alone."""
    cfg, _, model = _tiny(dtype)
    K, lens = cfg.num_codebooks, [0, 1, 3, 9, 5, 0]
    enc, em, prompt, pm = _inputs(cfg, 6, 8, 4, seed=3, dtype=dtype)
    codes, mask = _ragged_codes(cfg, lens, seed=4)
    kw = dict(max_new_tokens=14, do_sample=False, _suppress_special=mode == "greedy")
    if mode != "greedy":
        kw.update(_SAMPLED, output_scores=True, output_logits=True)
    if mode == "forced_bos":
        kw.update(forced_bos_token_id=3, begin_suppress_tokens=[3, 7])
    got = _generate(model, enc, em, prompt, pm, decoder_input_ids=codes, decoder_attention_mask=mask, **kw)
    assert got.raw_ids.shape[0] == 6 * K and len(got.audios_length) == 6
    for b in range(6):
        alone = _alone(model, enc, em, prompt, pm, codes, lens, b, **kw)
        _assert_row_equals_alone(got, alone, b, K, mode)
        assert torch.equal(got.audio_codes[b, :, :lens[b]], codes[b, :, :lens[b]])   # each row begins with its own prefix
        if mode != "greedy":
            _assert_steps_equal(got, alone, b, K, mode)


def _set_path(monkeypatch, mode):
    monkeypatch.delenv("PTTS_STEP", raising=False)
    monkeypatch.delenv("PTTS_FUSED", raising=False)
    if mode == "legacy":
        monkeypatch.setenv("PTTS_STEP", "legacy")
    if mode == "multi":
        monkeypatch.setenv("PTTS_FUSED", "0")


@pytest.mark.gpu
def test_mini_bf16_b32_paths_agree_and_rows_equal_alone(monkeypatch):
    """Mini bf16, 32 rows with prefixes spread over 0 .. 430 frames, top-k sampling: the cluster kernel, step.cu and the
    multi-kernel graph give the same ids and codes, and rows 0, 7 and 31 equal their alone runs."""
    cfg, _, model = _mini()
    K, B, S = cfg.num_codebooks, 32, 24
    lens = [(b * 431) // (B - 1) if b % 2 == 0 else (b * 137) % 431 for b in range(B)]
    lens[7], lens[16] = 250, 4
    enc, em, _, _ = _inputs(cfg, B, S, 0, seed=5, dtype=torch.bfloat16)
    codes, mask = _ragged_codes(cfg, lens, seed=6)
    kw = dict(do_sample=True, top_k=50, seed=9, max_new_tokens=16, return_codes=True)
    results = {}
    for mode in ("cluster", "legacy", "multi"):
        _set_path(monkeypatch, mode)
        results[mode] = _generate(model, enc, em, None, None, decoder_input_ids=codes, decoder_attention_mask=mask, **kw)
        assert model.decoder.engine._sessions[(B, 0, S)].fused == {"cluster": 2, "legacy": 1, "multi": 0}[mode]
    for mode in ("legacy", "multi"):
        assert torch.equal(results[mode].raw_ids, results["cluster"].raw_ids), mode
        assert torch.equal(results[mode].audio_codes, results["cluster"].audio_codes), mode
    # Rows against a batch of the same 32 rows that all continue from the row's own prefix (the bf16 prefill GEMM is picked by
    # its row count, B * (P + n0): a batch of one, or 32 rows of one column, take the other kernel and other last bits)
    _set_path(monkeypatch, "cluster")
    for b in (7, 16, 31):
        same = codes[b:b + 1, :, :lens[b]].expand(B, -1, -1).contiguous()
        ref = _generate(model, enc, em, None, None, decoder_input_ids=same, **kw)
        T = ref.raw_ids.shape[1]
        assert torch.equal(results["cluster"].raw_ids[b * K:(b + 1) * K, :T], ref.raw_ids[b * K:(b + 1) * K]), b
        F = ref.audio_codes.shape[-1]
        assert torch.equal(results["cluster"].audio_codes[b, :, :F], ref.audio_codes[b]), b


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["rope", "gqa"])
def test_mini_rope_and_gqa_on_step_kernel(monkeypatch, variant):
    """A rope checkpoint and a GQA one on step.cu (PTTS_STEP=legacy): rows equal their alone runs and the multi-kernel path."""
    kw_cfg = dict(rope_embeddings=True) if variant == "rope" else dict(num_key_value_heads=4)
    cfg, _, model = _mini(**kw_cfg)
    K, B, S = cfg.num_codebooks, 8, 16
    lens = [0, 40, 7, 120, 1, 64, 119, 3]
    enc, em, _, _ = _inputs(cfg, B, S, 0, seed=7, dtype=torch.bfloat16)
    codes, mask = _ragged_codes(cfg, lens, seed=8)
    kw = dict(max_new_tokens=12, return_codes=True, _suppress_special=True)
    _set_path(monkeypatch, "legacy")
    got = _generate(model, enc, em, None, None, decoder_input_ids=codes, decoder_attention_mask=mask, **kw)
    assert model.decoder.engine._sessions[(B, 0, S)].fused == 1
    for b in (3, 6):   # rows against a same-size batch of the row's own prefix (see the B = 32 test)
        ref = _generate(model, enc, em, None, None, decoder_input_ids=codes[b:b + 1, :, :lens[b]].expand(B, -1, -1).contiguous(), **kw)
        T = ref.raw_ids.shape[1]
        assert torch.equal(got.raw_ids[b * K:(b + 1) * K, :T], ref.raw_ids[b * K:(b + 1) * K]), b
    _set_path(monkeypatch, "multi")
    ref = _generate(model, enc, em, None, None, decoder_input_ids=codes, decoder_attention_mask=mask, **kw)
    assert torch.equal(got.raw_ids, ref.raw_ids)


@pytest.mark.gpu
def test_fp32_greedy_rows_against_the_oracle():
    """fp32 greedy: each row of a ragged call against the CPU oracle run on the row alone (tests/continuation_oracle.py): logits at
    the prefill and at every later step within 2e-4, ids exact -- generate()'s raw_ids are the history with the row's delay
    pattern applied (the prefix cells and the closing PAD cells), its codes the free cells of that."""
    import numpy as np
    from oracle.decoder import OracleDecoder
    from tests import continuation_oracle as co
    cfg, w, model = _tiny(torch.float32)
    K, B, S, P, M = cfg.num_codebooks, 4, 8, 4, 10
    lens = [6, 0, 2, 5]
    enc, em, prompt, pm = _inputs(cfg, B, S, P, seed=11, dtype=torch.float32)
    codes, mask = _ragged_codes(cfg, lens, seed=12)
    got = _generate(model, enc, em, prompt, pm, decoder_input_ids=codes, decoder_attention_mask=mask, max_new_tokens=M,
                    do_sample=False, output_logits=True)
    dec = OracleDecoder(cfg, w, torch.float32)
    for b in range(B):
        cpu = lambda t: t[b:b + 1].cpu()
        dii = None if lens[b] == 0 else codes[b, :, :lens[b]].cpu().numpy()
        ref = co.generate_tokens(dec, cfg, cpu(enc), cpu(em), cpu(prompt), cpu(pm), dict(max_new_tokens=M, do_sample=False),
                                 decoder_input_ids=dii, collect_logits=True)
        T = ref["raw_ids"].shape[1]
        assert ref["n0"] == lens[b] + 1 and T > ref["n0"]
        assert np.array_equal(got.raw_ids[b * K:(b + 1) * K, :T].cpu().numpy(),
                              co.apply_delay_pattern_mask(ref["raw_ids"], ref["delay_mask"])), b
        want = co.codes_from_raw(ref["raw_ids"], ref["input_ids"], cfg, 1, ref["max_length"])[0]
        assert np.array_equal(got.audio_codes[b, :, :want.shape[-1]].cpu().numpy(), want), b
        for t, lg in enumerate(ref["logits"]):
            err = float(np.abs(got.logits[t][b * K:(b + 1) * K].cpu().numpy() - np.asarray(lg).reshape(K, -1)).max())
            assert err < 2e-4, (b, t, err)


@pytest.mark.gpu
def test_begin_ids2_with_one_column_on_a_bos_only_session():
    """ptts_generate_begin_ids2 with n0 = 1 (every length 1, every offset 0) on a session without a continuation capacity
    (max_input_len = 1, no offset region): the uniform batch, the same history and tokens as ptts_generate_begin_ids."""
    cfg, _, model = _tiny(torch.float32)
    K, B, S, P, L = cfg.num_codebooks, 3, 8, 4, 12
    enc, em, prompt, pm = _inputs(cfg, B, S, P, seed=21, dtype=torch.float32)
    bos = torch.full((B * K, 1), cfg.bos_token_id, dtype=torch.long, device=DEV)
    runs = []
    for lens in (None, torch.ones(B, dtype=torch.int32, device=DEV)):
        sess = model.decoder.engine.session(B, P, S, P + L, max_input_len=1)
        sess.begin(L, do_sample=True, top_k=20, seed=4, input_ids=bos, input_lens=lens)
        sess.prefill(prompt, pm, enc, em)
        sess.sample()
        sess.decode_steps(L - 2)
        torch.cuda.synchronize()
        runs.append(sess.raw_ids[:, :int(sess.state[0].item())].clone())
    assert torch.equal(runs[0], runs[1])


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["cluster", "multi"])
def test_all_ones_mask_is_todays_result(monkeypatch, mode):
    """A mask of all ones gives the result without a mask bit for bit, on the same decode path."""
    _set_path(monkeypatch, mode)
    cfg, _, model = _mini()
    B, S, N = 4, 16, 12
    enc, em, _, _ = _inputs(cfg, B, S, 0, seed=13, dtype=torch.bfloat16)
    codes, mask = _ragged_codes(cfg, [N] * B, seed=14)
    kw = dict(do_sample=True, top_k=50, seed=2, max_new_tokens=10, output_scores=True)
    want = _generate(model, enc, em, None, None, decoder_input_ids=codes, **kw)
    path = model.decoder.engine._sessions[(B, 0, S)].fused
    got = _generate(model, enc, em, None, None, decoder_input_ids=codes, decoder_attention_mask=mask, **kw)
    assert model.decoder.engine._sessions[(B, 0, S)].fused == path == {"cluster": 2, "multi": 0}[mode]
    for k in ("raw_ids", "audio_codes", "sequences"):
        assert torch.equal(got[k], want[k]), k
    assert got.audios_length == want.audios_length
    for a, b in zip(got.scores, want.scores):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_takes_and_shards_equal_the_expanded_batch():
    """num_return_sequences = 3 over 15 descriptions (45 rows: shards of 30 + 15), ragged: equals the hand-expanded batch (its
    shards of 32 + 13), with the per-step scores of each row."""
    cfg, _, model = _mini()
    K, B, N, S = cfg.num_codebooks, 15, 3, 16
    lens = [(b * 7) % 23 for b in range(B)]
    enc, em, _, _ = _inputs(cfg, B, S, 0, seed=15, dtype=torch.bfloat16)
    codes, mask = _ragged_codes(cfg, lens, seed=16)
    kw = dict(do_sample=True, top_k=50, seed=4, max_new_tokens=10, output_scores=True)
    got = _generate(model, enc, em, None, None, decoder_input_ids=codes, decoder_attention_mask=mask, num_return_sequences=N, **kw)
    rep = lambda t: t.repeat_interleave(N, dim=0)
    want = _generate(model, rep(enc), rep(em), None, None, decoder_input_ids=rep(codes), decoder_attention_mask=rep(mask), **kw)
    for k in ("raw_ids", "audio_codes", "sequences"):
        assert torch.equal(got[k], want[k]), k
    assert got.audios_length == want.audios_length
    assert len(got.scores) == len(want.scores)
    for a, b in zip(got.scores, want.scores):
        assert torch.equal(torch.nan_to_num(a, nan=1e9), torch.nan_to_num(b, nan=1e9))


@pytest.mark.gpu
def test_input_values_list_equals_codes_of_each_clip():
    """input_values as a list of clips of different lengths continues exactly as decoder_input_ids holding each clip's own
    DACModel.encode codes, with the mask of their frame counts."""
    from parler_tts_b200 import ParlerTTSConfig, ParlerTTSForConditionalGeneration
    from oracle.weights import make_decoder_weights
    from tests.golden.make_dac_encode_golden import encode_cfg, weights
    from tests.helpers import product_decoder_config, synth_inputs
    from tests.test_dac_encode import product_codec_config
    cfg, dcfg = tiny_cfg(), encode_cfg()
    pc = ParlerTTSConfig(vocab_size=cfg.text_vocab_size, text_encoder={}, audio_encoder=product_codec_config(dcfg),
                         decoder=product_decoder_config(cfg))
    model = ParlerTTSForConditionalGeneration(pc, device=DEV, dtype=torch.bfloat16)
    model.load_state_dict(make_decoder_weights(cfg, seed=13, head_std=0.5), dac_state_dict=weights(dcfg))
    K, B = cfg.num_codebooks, 3
    g = torch.Generator().manual_seed(17)
    clips = [(0.3 * torch.randn(1, n, generator=g)).to(DEV) for n in (3 * 512 + 100, 7 * 512, 5 * 512 + 7)]
    clips[1] = clips[1][0]   # [samples] is taken too
    enc, em, _, _ = synth_inputs(cfg, B, 6, 0, seed=18)
    kw = dict(encoder_outputs=(enc.to(DEV),), attention_mask=em.to(DEV), max_new_tokens=10, return_dict_in_generate=True,
              do_sample=True, top_k=8, seed=3)
    got = model.generate(input_values=clips, **kw)
    own = [model.audio_encoder.encode(c.reshape(1, 1, -1)).audio_codes.reshape(K, -1) for c in clips]
    lens = [c.shape[-1] for c in own]
    codes = torch.zeros(B, K, max(lens), dtype=torch.long, device=DEV)
    for b, c in enumerate(own):
        codes[b, :, :lens[b]] = c
    mask = (torch.arange(max(lens))[None, :] < torch.tensor(lens)[:, None]).long().to(DEV)
    want = model.generate(decoder_input_ids=codes, decoder_attention_mask=mask, **kw)
    for k in ("raw_ids", "audio_codes", "sequences"):
        assert torch.equal(got[k], want[k]), k
    assert got.audios_length == want.audios_length
    for b in range(B):
        assert torch.equal(got.audio_codes[b, :, :lens[b]], own[b])
