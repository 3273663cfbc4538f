"""generate(decoder_input_ids=...): continuing from audio codes (modeling_parler_tts.py:2988-3046, :3442-3600).

Host tests pin the integer semantics (BOS column, generated length, delay pattern of the input, de-delay of the output) against
tests/golden/continuation.npz, which the reference's own code wrote, and check the shim's input validation.  GPU tests run the
device loop: fp32 against the CPU oracle, a generation continued from its own first frames, the decode paths bit for bit, batch
shards, the streamer and the returned codes.
"""
import os

import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg
from oracle.delay_pattern import build_delay_pattern_mask
from tests import continuation_oracle as co

DEV = "cuda"


# ---- host: the integer semantics against the reference's code ------------------------------------------------------------------
def _cases(golden_dir):
    z = np.load(os.path.join(golden_dir, "continuation.npz"))
    bos, pad = (int(v) for v in z["tokens"])
    for ci in range(int(z["n"])):
        B, K, N, with_bos, mnt, ml = (int(v) for v in z[f"c{ci}_meta"])
        yield ci, z, bos, pad, B, K, (None if mnt < 0 else mnt), (None if ml < 0 else ml)


def test_oracle_reproduces_reference_continuation_fixture(golden_dir):
    for ci, z, bos, pad, B, K, mnt, ml in _cases(golden_dir):
        ids = co.bos_led(z[f"c{ci}_codes"], K, bos)
        assert np.array_equal(ids, z[f"c{ci}_input_ids"]), ci
        L = co.generated_length(ids.shape[1], mnt, ml if ml is not None else 2580)
        assert L == int(z[f"c{ci}_max_length"]), ci
        delayed, mask = build_delay_pattern_mask(ids, bos, pad, L, K)
        assert np.array_equal(delayed, z[f"c{ci}_delayed"]), ci
        assert np.array_equal(mask, z[f"c{ci}_mask"]), ci
        cfg = tiny_cfg(num_codebooks=K, bos_token_id=bos, pad_token_id=pad)
        assert np.array_equal(co.codes_from_raw(z[f"c{ci}_full"], ids, cfg, B, L), z[f"c{ci}_frames"]), ci


def test_shim_bos_column_matches_reference(golden_dir):
    from parler_tts_b200.modeling import prepare_decoder_input_ids
    for ci, z, bos, pad, B, K, mnt, ml in _cases(golden_dir):
        codes = torch.from_numpy(z[f"c{ci}_codes"])
        got = prepare_decoder_input_ids(codes, B, K, 96, bos, "cpu")
        assert np.array_equal(got.numpy(), z[f"c{ci}_input_ids"]), ci
        # [B, K, N] and [1, B, K, N] (generate(return_codes=True)'s audio_codes[None]) are the same input
        got3 = prepare_decoder_input_ids(codes.reshape(1, B, K, -1), B, K, 96, bos, "cpu")
        assert torch.equal(got, got3)


def test_shim_rejects_bad_decoder_input_ids():
    from parler_tts_b200.modeling import check_continuation_length, prepare_decoder_input_ids
    ok = torch.zeros(2 * 4, 3, dtype=torch.long)
    prepare_decoder_input_ids(ok, 2, 4, 96, 65, "cpu")
    with pytest.raises(ValueError, match="rows"):        # row count other than B*K
        prepare_decoder_input_ids(torch.zeros(7, 3, dtype=torch.long), 2, 4, 96, 65, "cpu")
    with pytest.raises(ValueError, match="rows"):
        prepare_decoder_input_ids(torch.zeros(3 * 4, 3, dtype=torch.long), 2, 4, 96, 65, "cpu")
    with pytest.raises(ValueError, match="vocab_size"):  # ids outside [0, vocab_size]
        prepare_decoder_input_ids(torch.full((8, 3), 97, dtype=torch.long), 2, 4, 96, 65, "cpu")
    with pytest.raises(ValueError, match="vocab_size"):
        prepare_decoder_input_ids(torch.full((8, 3), -1, dtype=torch.long), 2, 4, 96, 65, "cpu")
    prepare_decoder_input_ids(torch.full((8, 3), 96, dtype=torch.long), 2, 4, 96, 65, "cpu")   # vocab_size itself is a table row
    with pytest.raises(ValueError, match="integer"):
        prepare_decoder_input_ids(torch.zeros(8, 3), 2, 4, 96, 65, "cpu")
    check_continuation_length(4, 10, 5, 128)
    with pytest.raises(ValueError, match="leaves no new token"):   # n0 >= max_length
        check_continuation_length(5, 10, 5, 128)
    with pytest.raises(ValueError, match="max_position_embeddings"):   # P + max_length above the position table
        check_continuation_length(4, 100, 29, 128)


def test_shard_batch_splits_decoder_input_ids_by_codebook_groups():
    from parler_tts_b200.dist import shard_batch
    B, K = 5, 4
    enc = torch.arange(B)[:, None].expand(B, 3)
    dii = torch.arange(B * K)[:, None].expand(B * K, 6)
    parts = [shard_batch({"decoder_input_ids": dii, "encoder_outputs": enc}, r, 2) for r in range(2)]
    assert [p["encoder_outputs"].shape[0] for p in parts] == [3, 2]
    assert torch.equal(torch.cat([p["decoder_input_ids"] for p in parts]), dii)
    assert torch.equal(parts[1]["decoder_input_ids"][:, 0], torch.arange(3 * K, 5 * K))


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
def _tiny_model(cfg, seed, dtype=torch.float32, head_std=0.5):
    from oracle.weights import make_dac_weights, make_decoder_weights
    from tests.helpers import build_product_model
    w = make_decoder_weights(cfg, seed=seed, head_std=head_std)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    return w, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=dtype)


def _prefix(cfg, B, N, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, cfg.codebook_size, (B * cfg.num_codebooks, N), generator=g)


def _session_run(model, enc, enc_mask, prompt, prompt_mask, input_ids, L):
    """begin(input_ids) + prefill + sample / decode_forward column by column: every step's logits and the raw history."""
    B, S, _ = enc.shape
    P = 0 if prompt is None else prompt.shape[1]
    n0 = input_ids.shape[1]
    sess = model.decoder.engine.session(B, P, S, P + L, max_input_len=n0)
    sess.begin(L, do_sample=False, input_ids=input_ids.to(DEV))
    sess.prefill(None if prompt is None else prompt.to(DEV), prompt_mask, enc.to(DEV), enc_mask)
    logits = [sess.logits.cpu().numpy().copy()]
    for c in range(n0, L):
        sess.sample()
        if c + 1 < L:
            sess.decode_forward()
            logits.append(sess.logits.cpu().numpy().copy())
    torch.cuda.synchronize()
    return logits, sess.raw_ids[:, :L].cpu().numpy().copy()


@pytest.mark.gpu
@pytest.mark.parametrize("N,P,mp", [(1, 4, 128), (4, 4, 128), (39, 4, 128), (2049, 8, 2304)])
def test_fp32_continuation_matches_oracle(N, P, mp):
    """fp32, greedy: logits at the prefill and at every later step within 2e-4, token ids bit-exact, with n0 = N + 1 input columns
    (the largest puts P + n0 = 2058 rows through the prefill)."""
    from oracle.decoder import OracleDecoder
    from tests.helpers import synth_inputs
    cfg = tiny_cfg(max_position_embeddings=mp)
    w, model = _tiny_model(cfg, seed=91)
    B, S = 2, 8
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=4)
    codes = _prefix(cfg, B, N, seed=N)
    L = N + 1 + 12
    dec = OracleDecoder(cfg, w, torch.float32)
    ref = co.generate_tokens(dec, cfg, enc, enc_mask, prompt, prompt_mask, dict(max_length=L, do_sample=False), codes.numpy(),
                             collect_logits=True)
    input_ids = torch.from_numpy(ref["input_ids"])
    logits, raw = _session_run(model, enc, enc_mask.to(DEV), prompt, prompt_mask.to(DEV), input_ids, L)
    n = ref["raw_ids"].shape[1]
    assert np.array_equal(raw[:, :n], ref["raw_ids"])
    for t in range(min(len(logits), len(ref["logits"]))):
        err = np.abs(logits[t] - ref["logits"][t]).max()
        assert err < 2e-4, (t, err)
    # generate(): same tokens, and the returned codes begin with the prefix frames
    _, out = model.generate(encoder_outputs=(enc.to(DEV),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV),
                            prompt_attention_mask=prompt_mask.to(DEV), decoder_input_ids=codes.to(DEV), do_sample=False,
                            max_length=L, return_codes=True)
    want = co.codes_from_raw(ref["raw_ids"], ref["input_ids"], cfg, B, L)
    assert np.array_equal(out.audio_codes.cpu().numpy(), want)
    assert np.array_equal(out.audio_codes[:, :, :N].cpu().numpy(), codes.reshape(B, cfg.num_codebooks, N).numpy())


@pytest.mark.gpu
def test_fp32_continuation_matches_oracle_mini_shape():
    from oracle.decoder import OracleDecoder
    from tests.helpers import synth_inputs
    cfg = mini_cfg(max_position_embeddings=256)
    w, model = _tiny_model(cfg, seed=71, head_std=0.2)
    B, S, P, N = 1, 12, 6, 30
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=5)
    codes = _prefix(cfg, B, N, seed=3)
    L = N + 1 + 10
    dec = OracleDecoder(cfg, w, torch.float32)
    ref = co.generate_tokens(dec, cfg, enc, enc_mask, prompt, prompt_mask, dict(max_length=L, do_sample=False), codes.numpy(),
                             collect_logits=True)
    logits, raw = _session_run(model, enc, enc_mask.to(DEV), prompt, prompt_mask.to(DEV), torch.from_numpy(ref["input_ids"]), L)
    n = ref["raw_ids"].shape[1]
    assert np.array_equal(raw[:, :n], ref["raw_ids"])
    for t in range(min(len(logits), len(ref["logits"]))):
        assert np.abs(logits[t] - ref["logits"][t]).max() < 2e-4, t


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 3, 9])
def test_continuing_from_own_frames_gives_the_same_tokens(m):
    """Generate without a prefix, then continue from the first m frames of that output: the later frames are the same (the
    decoder sees the same inputs at every position), apart from columns where the oracle's top-2 margin is below 2e-4."""
    from oracle.decoder import OracleDecoder
    from oracle.sampling import generate_tokens
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    w, model = _tiny_model(cfg, seed=93)
    B, S, P, L = 2, 8, 3, 40
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=6)
    kw = dict(encoder_outputs=(enc.to(DEV),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV),
              prompt_attention_mask=prompt_mask.to(DEV), do_sample=False, max_length=L, return_codes=True)
    _, first = model.generate(**kw)
    codes = first.audio_codes                                  # [B, K, T]
    _, cont = model.generate(decoder_input_ids=codes[:, :, :m].contiguous(), **kw)
    a, b = codes.cpu().numpy(), cont.audio_codes.cpu().numpy()
    # first column whose oracle margin is below 2e-4 (a near tie the two histories may break differently)
    ref = generate_tokens(OracleDecoder(cfg, w, torch.float32), cfg, enc, enc_mask, prompt, prompt_mask,
                          dict(max_length=L, do_sample=False), collect_logits=True)
    tie = len(ref["scores"])
    for t, s in enumerate(ref["scores"]):
        top = np.sort(s, axis=-1)[:, -2:]
        fin = np.isfinite(top).all(axis=-1)
        if (fin & (top[:, 1] - top[:, 0] < 2e-4)).any():
            tie = t
            break
    frames = min(a.shape[-1], b.shape[-1], max(0, tie + 1 - cfg.num_codebooks))   # column c -> frames up to c - K
    assert frames > m
    assert np.array_equal(a[..., :frames], b[..., :frames])
    assert np.array_equal(b[..., :m], a[..., :m])


def _mini_bf16_model():
    from oracle.weights import make_dac_weights, make_decoder_weights
    from tests.helpers import build_product_model
    cfg = mini_cfg()
    w = make_decoder_weights(cfg, seed=21, head_std=0.3)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    return cfg, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16)


def _mini_run(model, cfg, inputs, input_ids, L, gen, per_call=None):
    enc, enc_mask, prompt, prompt_mask = inputs
    B, S, _ = enc.shape
    P = prompt.shape[1]
    n0 = input_ids.shape[1]
    sess = model.decoder.engine.session(B, P, S, P + L, max_input_len=n0)
    sess.begin(L, min_new_tokens=L, suppress_special=True, codebook_size=cfg.codebook_size, seed=9, input_ids=input_ids, **gen)
    sess.prefill(prompt, prompt_mask, enc, enc_mask)
    logits = [sess.logits.cpu().numpy().copy()]
    sess.sample()
    left = L - n0 - 1
    while left > 0:
        n = left if per_call is None else min(per_call, left)
        sess.decode_steps(n)
        left -= n
        logits.append(sess.logits.cpu().numpy().copy())
    torch.cuda.synchronize()
    return sess.fused, sess.raw_ids[:, :L].cpu().numpy().copy(), logits


@pytest.mark.gpu
@pytest.mark.parametrize("gen", [dict(do_sample=False), dict(do_sample=True, top_k=50)], ids=["greedy", "topk50"])
def test_mini_bf16_batch32_paths_agree_with_a_430_frame_prefix(monkeypatch, gen):
    """Mini, bf16, B = 32, n0 = 431: the cluster kernel, PTTS_STEP=legacy and PTTS_FUSED=0 give identical ids and logits, and the
    cluster kernel gives the same for any number of steps per launch."""
    from tests.helpers import synth_inputs
    cfg, model = _mini_bf16_model()
    B, S, P, N = 32, 24, 16, 430
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=12)
    inputs = (enc.to(DEV).bfloat16(), enc_mask.to(DEV), prompt.to(DEV).bfloat16(), prompt_mask.to(DEV))
    from parler_tts_b200.modeling import prepare_decoder_input_ids
    ids = prepare_decoder_input_ids(_prefix(cfg, B, N, seed=8), B, cfg.num_codebooks, cfg.vocab_size, cfg.bos_token_id, DEV)
    L = N + 1 + 40
    runs = {}
    for mode in ("cluster", "legacy", "multi"):
        monkeypatch.delenv("PTTS_STEP", raising=False)
        monkeypatch.delenv("PTTS_FUSED", raising=False)
        if mode == "legacy":
            monkeypatch.setenv("PTTS_STEP", "legacy")
        if mode == "multi":
            monkeypatch.setenv("PTTS_FUSED", "0")
        runs[mode] = _mini_run(model, cfg, inputs, ids, L, gen, per_call=8)
    monkeypatch.delenv("PTTS_STEP", raising=False)
    monkeypatch.delenv("PTTS_FUSED", raising=False)
    for per_launch in ("1", "7"):
        monkeypatch.setenv("PTTS_STEPS_PER_LAUNCH", per_launch)
        runs["cluster/" + per_launch] = _mini_run(model, cfg, inputs, ids, L, gen, per_call=8)
    monkeypatch.delenv("PTTS_STEPS_PER_LAUNCH", raising=False)
    runs["cluster/one-call"] = _mini_run(model, cfg, inputs, ids, L, gen)
    assert runs["legacy"][0] == 1 and runs["multi"][0] == 0
    base = runs["legacy"]
    for name, (fused, raw, logits) in runs.items():
        if name.startswith("cluster") and fused != 2:
            continue   # the cluster kernel's grid does not fit this device
        assert np.array_equal(raw, base[1]), name
        if name != "cluster/one-call":
            assert all(np.array_equal(a, b) for a, b in zip(logits, base[2])), name
        else:
            assert np.array_equal(logits[-1], base[2][-1]), name


@pytest.mark.gpu
def test_batch_of_40_with_a_prefix_equals_its_shards():
    """bf16 above 32 rows runs as shards of <= 32 utterances, each with its K-row groups of the prefix: the result equals two
    separate calls (32 + 8, the second with row_base = 32 K) for greedy and top-k sampling."""
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    _, model = _tiny_model(cfg, seed=95, dtype=torch.bfloat16)
    B, S, P, N, L = 40, 8, 4, 6, 30
    K = cfg.num_codebooks
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=7)
    codes = _prefix(cfg, B, N, seed=5).to(DEV)
    for gen in (dict(do_sample=False), dict(do_sample=True, top_k=20, seed=3)):
        def run(lo, hi, row_base):
            _, out = model.generate(encoder_outputs=(enc[lo:hi].to(DEV),), attention_mask=enc_mask[lo:hi].to(DEV),
                                    prompt_hidden_states=prompt[lo:hi].to(DEV), prompt_attention_mask=prompt_mask[lo:hi].to(DEV),
                                    decoder_input_ids=codes[lo * K:hi * K], max_length=L, return_codes=True, row_base=row_base,
                                    _suppress_special=True, **gen)
            return out.audio_codes.cpu()
        whole = run(0, B, 0)
        parts = torch.cat([run(0, 32, 0), run(32, B, 32 * K)], dim=0)
        assert torch.equal(whole, parts), gen
        assert torch.equal(whole[:, :, :N], codes.cpu().reshape(B, K, N))


@pytest.mark.gpu
@pytest.mark.parametrize("B,incremental", [(1, False), (4, True)])
def test_streamer_with_a_prefix_equals_generate(B, incremental):
    from parler_tts_b200 import ParlerTTSStreamer
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    _, model = _tiny_model(cfg, seed=61)
    enc, _, prompt, _ = synth_inputs(cfg, B, 6, 3, seed=9, masks=False)
    codes = _prefix(cfg, B, 11, seed=2).to(DEV)
    kw = dict(encoder_outputs=(enc.to(DEV),), prompt_hidden_states=prompt.to(DEV), decoder_input_ids=codes, do_sample=False,
              max_length=50, _suppress_special=True)
    st = ParlerTTSStreamer(model, device=DEV, play_steps=6, incremental=incremental)
    audio = model.generate(streamer=st, **kw)
    chunks = [c for c in st]
    total = np.concatenate(chunks, axis=-1)
    full = audio.float().cpu().numpy()
    full = full[0] if B == 1 else full
    assert total.shape == full.shape and sum(c.shape[-1] > 0 for c in chunks) >= 2
    if incremental:   # every emitted sample is final; the reference mode re-decodes the history and emits provisional samples
        assert np.abs(total - full).max() < 1e-4
    assert np.abs(model.generate(**kw).float().cpu().numpy() - audio.float().cpu().numpy()).max() == 0.0   # the streamer changes nothing
