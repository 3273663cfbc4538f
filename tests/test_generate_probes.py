"""output_attentions / output_hidden_states: generate(), forward() and the step operator.

Host tests: the GenerationConfig fields, the recorder's chunk arithmetic and the probe oracle's eager definition.  GPU tests: the
attention-weights kernel against an fp64 restatement (ptts_op_attention_probs), generate() and forward() against the oracle, and
tokens / scores / waveform bit-identical with and without the flags on the cluster kernel, in shards, with a streamer and on
the host-driven loop.
"""
import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg

DEV = "cuda"
PROBE = dict(return_dict_in_generate=True, output_attentions=True, output_hidden_states=True)


# ---- host ----------------------------------------------------------------------------------------------------------------------
def test_generation_config_probe_fields_default_off():
    from parler_tts_b200 import GenerationConfig
    gc = GenerationConfig()
    assert gc.output_attentions is False and gc.output_hidden_states is False
    assert gc.update(output_attentions=True, output_hidden_states=True) == {}
    assert gc.output_attentions is True and gc.output_hidden_states is True


def test_step_probes_entries_and_chunks():
    from parler_tts_b200.modeling import StepProbes
    p = StepProbes(n_layers=2, batch=3, heads=4, S=5, H=8, P=6, n0=2, dtype=torch.float32, device="cpu", attentions=True, hidden=True)
    assert p.t_hi(0) == 6 + 2 + 63 and p.t_hi(2) == 6 + 2 + 191
    assert p.chunks == {}
    e0 = p.entry(0)
    assert [t.shape for t in e0["decoder_attentions"]] == [(3, 4, 8, 8)] * 2
    assert [t.shape for t in e0["cross_attentions"]] == [(3, 4, 8, 5)] * 2
    assert [t.shape for t in e0["decoder_hidden_states"]] == [(3, 8, 8)] * 3
    e = p.entry(130)                       # allocates chunk 2 only
    assert list(p.chunks) == [2]
    assert [t.shape for t in e["decoder_attentions"]] == [(3, 4, 1, 6 + 2 + 130)] * 2
    assert [t.shape for t in e["cross_attentions"]] == [(3, 4, 1, 5)] * 2
    assert [t.shape for t in e["decoder_hidden_states"]] == [(3, 1, 8)] * 3
    assert torch.isnan(e["decoder_attentions"][0]).all()
    r = p.result(3)
    assert set(r) == {"decoder_attentions", "cross_attentions", "decoder_hidden_states"} and len(r["decoder_attentions"]) == 3
    q = StepProbes(2, 3, 4, 5, 8, 6, 2, torch.float32, "cpu", attentions=False, hidden=True)
    assert set(q.result(2)) == {"decoder_hidden_states"}


def test_eager_weights_definition():
    from tests.probe_oracle import eager_weights
    g = torch.Generator().manual_seed(0)
    qs, ks = torch.randn(2, 3, 4, 64, generator=g), torch.randn(2, 3, 6, 64, generator=g)
    m = torch.zeros(2, 1, 4, 6, dtype=torch.bool)
    m[0, 0, :, 1] = True
    m[1, 0, 2, :] = True                   # a row with every key masked: uniform
    for dt in (torch.float32, torch.bfloat16):
        w = eager_weights(qs, ks, m, dt)
        assert w.dtype == dt
        assert (w[0, :, :, 1] == 0).all()
        assert torch.allclose(w[1, :, 2].float(), torch.full((3, 6), 1 / 6), atol=1e-3)
        assert torch.allclose(w.float().sum(-1), torch.ones(2, 3, 4), atol=2e-2)
        s = (qs.to(dt) * 0.125).to(dt) @ ks.to(dt).transpose(2, 3)
        ref = torch.softmax(s.float().masked_fill(m, -float("inf")), -1)
        ok = ~m.expand(2, 3, 4, 6) & ~m.all(-1, keepdim=True).expand(2, 3, 4, 6)
        assert torch.allclose(w.float()[ok], ref[ok].to(dt).float())


GOLDEN_CASES = {   # tests/golden/make_probes_golden.py CASES: tiny_cfg overrides, weight seed
    "sin": (dict(), 31),
    "rope": (dict(rope_embeddings=True), 32),
    "rope_gqa": (dict(rope_embeddings=True, hidden_size=256, num_attention_heads=4, num_key_value_heads=2,
                      num_cross_attention_key_value_heads=2), 33),
}


@pytest.mark.parametrize("case", list(GOLDEN_CASES))
def test_probe_oracle_reproduces_reference_fixture(golden_dir, case):
    """tests/golden/probes.npz: the reference's ParlerTTSForCausalLM.forward(use_cache=False, output_attentions=True,
    output_hidden_states=True) with eager attention (make_probes_golden.py).  The oracle every value test uses reproduces its
    attention weights and its L + 1 hidden states, in order, on every row the decoder computes for a later row to read."""
    import os
    from tests.probe_oracle import ProbeOracleDecoder
    from oracle.weights import make_decoder_weights
    z = np.load(os.path.join(golden_dir, "probes.npz"))
    over, seed = GOLDEN_CASES[case]
    cfg = tiny_cfg(**over)
    B, K, P, S, T, _ = (int(x) for x in z[f"{case}_meta"])
    pm = torch.from_numpy(z[f"{case}_pmask"])
    o = ProbeOracleDecoder(cfg, make_decoder_weights(cfg, seed=seed), torch.float32)
    o.prefill(torch.from_numpy(z[f"{case}_dec"]), torch.from_numpy(z[f"{case}_enc"]), torch.from_numpy(z[f"{case}_enc_mask"]),
              torch.from_numpy(z[f"{case}_prompt"]), pm)
    rec = o.calls[0]
    L = cfg.num_hidden_layers
    ref_self, ref_cross, ref_hidden = (torch.from_numpy(z[f"{case}_{k}"]) for k in ("self", "cross", "hidden"))
    assert ref_self.shape == (L, B, cfg.num_attention_heads, P + T, P + T) and ref_hidden.shape[0] == L + 1
    # layer 0 sees the same input on every row: all of its self-attention weights match, the fully masked rows included
    assert (rec["self"][0] - ref_self[0]).abs().max() <= 1e-5
    for l in range(L):
        assert (_live(rec["self"][l], pm, P, 2) - _live(ref_self[l], pm, P, 2)).abs().max() <= 1e-5, l
        assert (_live(rec["cross"][l], pm, P, 2) - _live(ref_cross[l], pm, P, 2)).abs().max() <= 1e-5, l
    for e in range(L + 1):
        ref = _live(ref_hidden[e], pm, P, 1)
        assert (_live(rec["hidden"][e], pm, P, 1) - ref).abs().max() <= 1e-4 * max(1.0, float(ref.abs().max())), e


# ---- GPU: the kernel against fp64 ----------------------------------------------------------------------------------------------
def _swizzle_rows(k):
    """[..., T, 64] rows -> their stored order (element d of row t at ((d/8 ^ t) % 8) * 8 + d % 8)."""
    T = k.shape[-2]
    out = torch.empty_like(k)
    t = torch.arange(T)[:, None]
    d = torch.arange(64)[None, :]
    pos = ((((d >> 3) ^ t) & 7) << 3) | (d & 7)
    out.scatter_(-1, pos.expand(*k.shape), k)
    return out


def _rope_ref(x, cos, sin, dt):
    """x [.., q, 64] in dt, the rotary step in the model dtype (every product and the sum rounded)."""
    rot = torch.cat((-x[..., 32:], x[..., :32]), dim=-1)
    return ((x * cos).to(dt) + (rot * sin).to(dt)).to(dt)


CASES = [  # B, nh, nkv, q_len, past, cross, kv_len, rope, mask_len
    (2, 4, 4, 1, 36, 0, 37, 0, 8),
    (2, 4, 2, 1, 4094, 0, 4095, 1, 16),
    (1, 4, 4, 37, 0, 0, 37, 1, 12),
    (1, 2, 1, 300, 3795, 0, 4095, 0, 40),
    (2, 4, 2, 9, 0, 1, 77, 1, 77),
    (3, 4, 4, 1, 0, 1, 33, 0, 33),
]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("case", CASES, ids=[f"B{c[0]}h{c[1]}kv{c[2]}q{c[3]}p{c[4]}{'x' if c[5] else 's'}{c[6]}r{c[7]}" for c in CASES])
def test_attention_probs_kernel_against_fp64(case, dtype):
    from parler_tts_b200 import _lib
    B, nh, nkv, q_len, past, cross, kv_len, rope, mask_len = case
    g = torch.Generator().manual_seed(sum(case))
    # small multiples of 1/8 (and rotary tables in {0, +-1/2, +-1}): every dot product is exact in fp32, so the rounded scores
    # are the fp64 ones and the tolerance is the rounding of the weights alone
    q = torch.randint(-3, 4, (B, q_len, nh, 64), generator=g).float() / 8
    k = torch.randint(-3, 4, (B, nkv, kv_len, 64), generator=g).float() / 8
    cap = kv_len + 5
    maxpos = past + q_len + 1
    cos = torch.randint(-2, 3, (maxpos, 64), generator=g).float() / 2
    sin = torch.randint(-2, 3, (maxpos, 64), generator=g).float() / 2
    km = (torch.rand(B, mask_len, generator=g) > 0.3).int()
    km[0, :] = 0                                             # row 0: every prompt position padded
    dt = dtype
    kc = torch.zeros(B, nkv, cap, 64)
    kc[:, :, :kv_len] = k
    kc = _swizzle_rows(kc).to(dt).to(DEV)
    out = torch.full((B, nh, q_len, kv_len), float("nan"), dtype=dt, device=DEV)
    qd = q.reshape(B * q_len, nh * 64).to(dt).to(DEV)
    cosd, sind = cos.to(dt).to(DEV), sin.to(dt).to(DEV)
    kmd = km.to(DEV)
    code = 0 if dt == torch.bfloat16 else 1
    _lib.check(_lib.lib().ptts_op_attention_probs(code, B, nh, nkv, q_len, past, cross, kv_len, cap, rope, _lib.ptr(cosd), _lib.ptr(sind),
                                                  _lib.ptr(qd), nh * 64, _lib.ptr(kc), _lib.ptr(kmd), mask_len, _lib.ptr(out),
                                                  _lib.stream_ptr()))
    torch.cuda.synchronize()
    got = out.float().cpu().double()
    # fp64 reference
    qh = q.to(dt).permute(0, 2, 1, 3)                        # [B, nh, q, 64]
    if rope:
        pos = torch.arange(past, past + q_len)
        qh = _rope_ref(qh, cos.to(dt)[pos], sin.to(dt)[pos], dt)
    qh = (qh * 0.125).to(dt).double()
    kh = k.to(dt).double().repeat_interleave(nh // nkv, dim=1)
    s = (qh @ kh.transpose(2, 3)).to(dt).double()
    m = torch.zeros(B, 1, q_len, kv_len, dtype=torch.bool)
    pad = torch.zeros(B, kv_len, dtype=torch.bool)
    pad[:, :min(mask_len, kv_len)] = km[:, :kv_len] == 0
    m |= pad[:, None, None, :]
    if not cross:
        m |= (torch.arange(kv_len)[None, :] > torch.arange(past, past + q_len)[:, None])[None, None]
    m = m.expand(B, nh, q_len, kv_len)
    full = m.all(-1, keepdim=True)
    p = torch.softmax(s.masked_fill(m, -float("inf")), -1)
    p = torch.where(full, torch.full_like(p, 1.0 / kv_len), torch.nan_to_num(p, nan=0.0))
    ulp = 2.0 ** -8 if dt == torch.bfloat16 else 2.0 ** -21
    assert torch.isfinite(got).all()
    err = (got - p).abs()
    assert (err <= ulp * p.abs() + 1e-30).all(), float((err - ulp * p.abs()).max())
    assert (got[m & ~full] == 0).all()
    sums = got.sum(-1)
    assert ((sums - 1).abs() <= kv_len * ulp / 2 + 1e-6).all()


# ---- GPU: generate() and forward() ---------------------------------------------------------------------------------------------
def _model(cfg, seed, dtype, head_std=0.5):
    from oracle.weights import make_dac_weights, make_decoder_weights
    from tests.helpers import build_product_model
    w = make_decoder_weights(cfg, seed=seed, head_std=head_std)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=min(cfg.codebook_size, cfg.vocab_size - 8))
    return w, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=dtype)


def _kw(inputs, dtype):
    enc, enc_mask, prompt, prompt_mask = inputs
    return dict(encoder_outputs=(enc.to(DEV).to(dtype),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV).to(dtype),
                prompt_attention_mask=prompt_mask.to(DEV))


def _live(x, prompt_mask, P, dim):
    """x with the rows of padded prompt positions zeroed (dim = the query dimension): their self-attention sees no key, so what
    the decoder computes there is never read by any other row, and the restated attention fills them differently from SDPA."""
    if prompt_mask is None or x.shape[dim] < P:
        return x.float().cpu()
    keep = torch.ones(x.shape[0], x.shape[dim], dtype=torch.bool)
    keep[:, :P] = prompt_mask.cpu() != 0
    shape = [x.shape[0]] + [1] * (x.dim() - 1)
    shape[dim] = x.shape[dim]
    return x.float().cpu() * keep.view(shape)


def _check_against_oracle(out, calls, cfg, B, P, n0, S, dtype, prompt_mask):
    L, nh, H = cfg.num_hidden_layers, cfg.num_attention_heads, cfg.hidden_size
    n = len(out.decoder_attentions)
    assert n == out.raw_ids.shape[1] - n0 == len(out.cross_attentions) == len(out.decoder_hidden_states) == len(calls)
    tol_w, tol_h = (2e-4, 2e-3) if dtype == torch.float32 else (3e-2, 6e-2)
    for t in range(n):
        q = P + n0 if t == 0 else 1
        T = P + n0 + t
        assert len(out.decoder_attentions[t]) == L and len(out.decoder_hidden_states[t]) == L + 1
        for l in range(L):
            sa, ca = out.decoder_attentions[t][l], out.cross_attentions[t][l]
            assert sa.shape == (B, nh, q, T) and ca.shape == (B, nh, q, S) and sa.dtype == dtype and ca.dtype == dtype
            assert (_live(sa, prompt_mask, P, 2) - _live(calls[t]["self"][l], prompt_mask, P, 2)).abs().max() <= tol_w, (t, l)
            assert (_live(ca, prompt_mask, P, 2) - _live(calls[t]["cross"][l], prompt_mask, P, 2)).abs().max() <= tol_w, (t, l)
        for e in range(L + 1):
            hs = out.decoder_hidden_states[t][e]
            ref = _live(calls[t]["hidden"][e], prompt_mask, P, 1)
            assert hs.shape == (B, q, H) and hs.dtype == dtype
            assert (_live(hs, prompt_mask, P, 1) - ref).abs().max() <= tol_h * max(1.0, float(ref.abs().max())), (t, e)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("prefix", [0, 5], ids=["bos", "continuation"])
def test_generate_probes_match_oracle_and_leave_tokens_alone(dtype, prefix):
    from tests import sampling_ext_oracle as so
    from tests.helpers import synth_inputs
    from tests.probe_oracle import ProbeOracleDecoder
    cfg = tiny_cfg(num_key_value_heads=2)
    w, model = _model(cfg, seed=13, dtype=dtype)
    B, S, P, Lmax = 3, 8, 4, 18
    inputs = synth_inputs(cfg, B, S, P, seed=4)
    kw = _kw(inputs, dtype)
    ids = None
    if prefix:
        g = np.random.default_rng(3)
        ids = np.concatenate([np.full((B * cfg.num_codebooks, 1), cfg.bos_token_id),
                              g.integers(0, 40, size=(B * cfg.num_codebooks, prefix))], axis=1).astype(np.int64)
        kw["decoder_input_ids"] = torch.from_numpy(ids).to(DEV)
    n0 = 1 if ids is None else ids.shape[1]
    base = model.generate(**kw, max_length=Lmax + n0, return_dict_in_generate=True, output_scores=True)
    out = model.generate(**kw, max_length=Lmax + n0, output_scores=True, **PROBE)
    assert torch.equal(out.raw_ids, base.raw_ids) and torch.equal(out.sequences, base.sequences)
    assert all(torch.equal(a, b) for a, b in zip(out.scores, base.scores))
    assert out.encoder_attentions is None and out.encoder_hidden_states is None
    hist = out.raw_ids.cpu().numpy()
    enc, enc_mask, prompt, prompt_mask = inputs
    dec = ProbeOracleDecoder(cfg, w, dtype)
    so.generate_tokens(dec, cfg, enc, enc_mask, prompt, prompt_mask, dict(max_length=Lmax + n0), decoder_input_ids=ids,
                       pick=lambda step, s: hist[:, n0 + step])
    _check_against_oracle(out, dec.calls, cfg, B, P, n0, S, dtype, prompt_mask)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16-fused-score"])
def test_forward_probes_match_oracle_and_leave_the_loss_alone(dtype):
    """bf16 with labels scores on the fused heads + cross-entropy kernel, which reads the residual stream after the probe kernels."""
    from tests.helpers import synth_inputs
    from tests.probe_oracle import ProbeOracleDecoder
    cfg = tiny_cfg(rope_embeddings=True, num_key_value_heads=2)
    w, model = _model(cfg, seed=17, dtype=dtype)
    B, S, P, T, K = 2, 8, 4, 10, cfg.num_codebooks
    inputs = synth_inputs(cfg, B, S, P, seed=6)
    g = torch.Generator().manual_seed(2)
    labels = torch.randint(0, 60, (B, T, K), generator=g)
    kw = _kw(inputs, dtype)
    base = model.forward(**kw, labels=labels.to(DEV))
    out = model.forward(**kw, labels=labels.to(DEV), output_attentions=True, output_hidden_states=True)
    assert torch.equal(out.loss, base.loss) and torch.equal(out.token_losses, base.token_losses)
    assert all(torch.equal(a, b) for a, b in zip(out.per_codebook_losses, base.per_codebook_losses))
    tol_w, tol_h = (2e-4, 2e-3) if dtype == torch.float32 else (3e-2, 6e-2)
    from parler_tts_b200.modeling import shift_tokens_right
    dec_ids = shift_tokens_right(labels, cfg.pad_token_id, cfg.bos_token_id).transpose(1, 2).reshape(B * K, T)
    enc, enc_mask, prompt, prompt_mask = inputs
    o = ProbeOracleDecoder(cfg, w, dtype)
    o.prefill(dec_ids, enc, enc_mask, prompt, prompt_mask)
    rec = o.calls[0]
    L = cfg.num_hidden_layers
    assert len(out.decoder_attentions) == L and len(out.decoder_hidden_states) == L + 1
    for l in range(L):
        assert out.decoder_attentions[l].shape == (B, cfg.num_attention_heads, P + T, P + T)
        assert out.cross_attentions[l].shape == (B, cfg.num_attention_heads, P + T, S)
        live = lambda x: _live(x, prompt_mask, P, 2)
        assert out.decoder_attentions[l].dtype == dtype
        assert (live(out.decoder_attentions[l]) - live(rec["self"][l])).abs().max() <= tol_w
        assert (live(out.cross_attentions[l]) - live(rec["cross"][l])).abs().max() <= tol_w
    for e in range(L + 1):
        ref = _live(rec["hidden"][e], prompt_mask, P, 1)
        assert (_live(out.decoder_hidden_states[e], prompt_mask, P, 1) - ref).abs().max() <= tol_h * max(1.0, float(ref.abs().max()))


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(GOLDEN_CASES))
def test_forward_probes_reproduce_reference_fixture(golden_dir, case):
    """forward(decoder_input_ids=..., output_attentions=True, output_hidden_states=True) against the reference's own eager
    outputs (tests/golden/probes.npz), fp32: sinusoidal positions, RoPE, and RoPE with grouped-query attention."""
    import os
    from oracle.weights import make_decoder_weights
    from tests.helpers import build_product_model
    from oracle.weights import make_dac_weights
    z = np.load(os.path.join(golden_dir, "probes.npz"))
    over, seed = GOLDEN_CASES[case]
    cfg = tiny_cfg(**over)
    w = make_decoder_weights(cfg, seed=seed)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=min(cfg.codebook_size, cfg.vocab_size - 8))
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.float32)
    B, K, P, S, T, _ = (int(x) for x in z[f"{case}_meta"])
    pm = torch.from_numpy(z[f"{case}_pmask"])
    t = lambda k: torch.from_numpy(z[f"{case}_{k}"]).to(DEV)
    out = model.forward(encoder_outputs=(t("enc"),), attention_mask=t("enc_mask"), prompt_hidden_states=t("prompt"),
                        prompt_attention_mask=t("pmask"), decoder_input_ids=t("dec"), output_attentions=True, output_hidden_states=True)
    L = cfg.num_hidden_layers
    ref_self, ref_cross, ref_hidden = (torch.from_numpy(z[f"{case}_{k}"]) for k in ("self", "cross", "hidden"))
    assert (out.decoder_attentions[0].cpu() - ref_self[0]).abs().max() <= 2e-4   # layer 0: every row, fully masked ones included
    for l in range(L):
        assert (_live(out.decoder_attentions[l], pm, P, 2) - _live(ref_self[l], pm, P, 2)).abs().max() <= 2e-4, l
        assert (_live(out.cross_attentions[l], pm, P, 2) - _live(ref_cross[l], pm, P, 2)).abs().max() <= 2e-4, l
    for e in range(L + 1):
        ref = _live(ref_hidden[e], pm, P, 1)
        assert (_live(out.decoder_hidden_states[e], pm, P, 1) - ref).abs().max() <= 2e-3 * max(1.0, float(ref.abs().max())), e


@pytest.mark.gpu
def test_step_operator_returns_its_step():
    from tests.helpers import synth_inputs
    from parler_tts_b200.modeling import ParlerTTSForCausalLM
    cfg = tiny_cfg()
    w, model = _model(cfg, seed=5, dtype=torch.float32)
    dec = model.decoder
    assert isinstance(dec, ParlerTTSForCausalLM)
    B, S, P, K = 2, 8, 4, cfg.num_codebooks
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, B, S, P, seed=1)
    bos = torch.full((B * K, 1), cfg.bos_token_id, dtype=torch.long, device=DEV)
    kw = dict(encoder_hidden_states=enc.to(DEV), encoder_attention_mask=enc_mask.to(DEV), prompt_hidden_states=prompt.to(DEV),
              prompt_attention_mask=prompt_mask.to(DEV), max_cache_len=P + 8)
    plain = dec(bos, **kw)
    r0 = dec(bos, **kw, output_attentions=True, output_hidden_states=True)
    assert torch.equal(r0.logits, plain.logits)
    assert [a.shape for a in r0.attentions] == [(B, cfg.num_attention_heads, P + 1, P + 1)] * cfg.num_hidden_layers
    assert [h.shape for h in r0.hidden_states] == [(B, P + 1, cfg.hidden_size)] * (cfg.num_hidden_layers + 1)
    nxt = r0.logits[:, 0].argmax(-1, keepdim=True)
    p1 = dec(nxt, past_key_values=plain.past_key_values)
    r1 = dec(nxt, past_key_values=r0.past_key_values, output_attentions=True)
    assert torch.equal(r1.logits, p1.logits)
    assert [a.shape for a in r1.attentions] == [(B, cfg.num_attention_heads, 1, P + 2)] * cfg.num_hidden_layers
    assert [a.shape for a in r1.cross_attentions] == [(B, cfg.num_attention_heads, 1, S)] * cfg.num_hidden_layers
    assert torch.allclose(r1.attentions[0].float().sum(-1), torch.ones(B, cfg.num_attention_heads, 1, device=DEV), atol=1e-5)
    # a decode step's entry holds its own rows only: one [B, L, heads, T_kv] block, nothing sized by a chunk of steps
    L, nh = cfg.num_hidden_layers, cfg.num_attention_heads
    assert r1.attentions[0].untyped_storage().nbytes() == B * L * nh * (P + 2) * 4
    assert r1.cross_attentions[0].untyped_storage().nbytes() == B * L * nh * S * 4
    # the values, against the oracle stepped the same way
    from tests.probe_oracle import ProbeOracleDecoder
    o = ProbeOracleDecoder(cfg, w, torch.float32)
    o.prefill(bos.cpu(), enc, enc_mask, prompt, prompt_mask)
    # the step's decoder input is the appended column under the delay pattern (codebooks k > 0 still read BOS at step 1)
    from parler_tts_b200.modeling import apply_delay_pattern_mask, build_delay_pattern_mask
    hist = r1.past_key_values.session.raw_ids[:, :2].clone()
    _, pmask = build_delay_pattern_mask(hist[:, :1], cfg.bos_token_id, cfg.pad_token_id, 8, K)
    o.step(apply_delay_pattern_mask(hist, pmask)[:, 1:2].cpu())
    for got, rec in ((r0, o.calls[0]), (r1, o.calls[1])):
        for l in range(L):
            assert (_live(got.attentions[l], prompt_mask, P, 2) - _live(rec["self"][l], prompt_mask, P, 2)).abs().max() <= 2e-4
            assert (_live(got.cross_attentions[l], prompt_mask, P, 2) - _live(rec["cross"][l], prompt_mask, P, 2)).abs().max() <= 2e-4
    for e in range(L + 1):
        ref = _live(o.calls[0]["hidden"][e], prompt_mask, P, 1)
        assert (_live(r0.hidden_states[e], prompt_mask, P, 1) - ref).abs().max() <= 2e-3 * max(1.0, float(ref.abs().max()))


# ---- GPU: nothing else moves ---------------------------------------------------------------------------------------------------
def _same_outputs(a, b):
    assert torch.equal(a.raw_ids, b.raw_ids)
    assert torch.equal(a.sequences, b.sequences)
    for k in ("scores", "logits"):
        if a.get(k) is not None:
            assert len(a[k]) == len(b[k])
            for x, y in zip(a[k], b[k]):
                assert torch.equal(torch.nan_to_num(x, nan=7.0), torch.nan_to_num(y, nan=7.0)), k


@pytest.mark.gpu
def test_mini_cluster_path_bit_identical_with_probes():
    cfg = mini_cfg(num_hidden_layers=4)
    _, model = _model(cfg, seed=21, dtype=torch.bfloat16, head_std=0.3)
    from tests.helpers import synth_inputs
    B, S, P = 32, 12, 6
    inputs = synth_inputs(cfg, B, S, P, seed=9)
    kw = _kw(inputs, torch.bfloat16)
    gen = dict(do_sample=True, temperature=0.9, top_k=50, max_length=40, seed=3, return_dict_in_generate=True, output_scores=True,
               output_logits=True)
    base = model.generate(**kw, **gen)
    sess = next(iter(model.decoder.engine._sessions.values()))
    fused, launches0 = sess.fused, sess.launches
    assert fused == 2   # the cluster kernel
    out = model.generate(**kw, **gen, output_attentions=True, output_hidden_states=True)
    _same_outputs(out, base)
    assert sess.fused == fused
    n = out.raw_ids.shape[1] - 1
    assert len(out.decoder_attentions) == n and out.decoder_attentions[n - 1][3].shape == (B, cfg.num_attention_heads, 1, P + n)
    assert torch.isfinite(out.decoder_attentions[n - 1][3].float()).all()
    # the flags off again: the same path, the same launches as the first call, nothing recorded
    l1 = sess.launches
    again = model.generate(**kw, **gen)
    _same_outputs(again, base)
    assert sess.fused == fused and sess.launches - l1 == launches0
    assert "decoder_attentions" not in again


@pytest.mark.gpu
def test_shards_streamer_and_host_loop_bit_identical_with_probes():
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=8, dtype=torch.bfloat16)
    B, S, P = 40, 8, 4
    inputs = synth_inputs(cfg, B, S, P, seed=2)
    kw = _kw(inputs, torch.bfloat16)
    gen = dict(do_sample=True, top_k=30, max_length=30, seed=11, return_dict_in_generate=True, output_scores=True)
    base = model.generate(**kw, **gen)
    out = model.generate(**kw, **gen, output_attentions=True, output_hidden_states=True)
    _same_outputs(out, base)
    n = out.raw_ids.shape[1] - 1
    assert out.decoder_attentions[n - 1][0].shape == (B, cfg.num_attention_heads, 1, P + n)
    # streamer and a user logits_processor (host-driven loop) on the first 4 utterances
    class Cols:
        def __init__(self):
            self.cols = []

        def put(self, v):
            self.cols.append(v.clone())

        def end(self):
            pass
    sub = {k: (v[:4] if isinstance(v, torch.Tensor) else (v[0][:4],)) for k, v in kw.items()}
    s0, s1 = Cols(), Cols()
    a = model.generate(**sub, **gen, streamer=s0)
    b = model.generate(**sub, **gen, streamer=s1, output_attentions=True, output_hidden_states=True)
    _same_outputs(a, b)
    assert len(s0.cols) == len(s1.cols) and all(torch.equal(x, y) for x, y in zip(s0.cols, s1.cols))
    assert len(b.decoder_hidden_states) == b.raw_ids.shape[1] - 1
    proc = [lambda ids, scores: scores]
    c = model.generate(**sub, **gen, logits_processor=proc)
    d = model.generate(**sub, **gen, logits_processor=proc, output_attentions=True)
    _same_outputs(c, d)
    nd = d.raw_ids.shape[1] - 1
    assert len(d.decoder_attentions) == nd and torch.isfinite(d.decoder_attentions[nd - 1][1].float()).all()


@pytest.mark.gpu
def test_flags_off_allocate_no_recorder(monkeypatch):
    """Calls without the flags (or with them but without return_dict_in_generate, as in transformers) never build a recorder."""
    from parler_tts_b200 import modeling
    from tests.helpers import synth_inputs
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=8, dtype=torch.bfloat16)
    kw = _kw(synth_inputs(cfg, 3, 8, 4, seed=2), torch.bfloat16)
    with_rec = model.generate(**kw, max_length=12, return_dict_in_generate=True)

    def refuse(*a, **k):
        raise AssertionError("a recorder was built for a call that did not ask for one")
    monkeypatch.setattr(modeling, "StepProbes", refuse)
    a = model.generate(**kw, max_length=12, return_dict_in_generate=True)
    b = model.generate(**kw, max_length=12, output_attentions=True, output_hidden_states=True)   # no dict return: nothing recorded
    assert torch.equal(a.raw_ids, with_rec.raw_ids) and torch.equal(b, a.sequences)
    assert "decoder_attentions" not in a
    labels = torch.randint(0, 60, (3, 5, cfg.num_codebooks)).to(DEV)
    model.forward(**kw, labels=labels)
    sess = next(iter(model.decoder.engine._sessions.values()))
    assert sess._probes is None


@pytest.mark.gpu
def test_encoder_outputs_from_generate_input_ids():
    """generate(input_ids=...) with the flags runs the text encoder eagerly with them and returns its tuples; the tokens are those
    of the graphed encoder call."""
    from transformers import T5Config, T5EncoderModel
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=12, dtype=torch.float32)
    tc = T5Config(vocab_size=128, d_model=cfg.hidden_size, d_kv=16, d_ff=128, num_layers=2, num_heads=4, dropout_rate=0.0)
    torch.manual_seed(0)
    model.text_encoder = T5EncoderModel(tc).to(DEV).eval()
    B, S = 2, 7
    ids = torch.randint(0, 128, (B, S)).to(DEV)
    am = torch.ones(B, S, dtype=torch.long, device=DEV)
    am[1, 5:] = 0
    base = model.generate(input_ids=ids, attention_mask=am, max_length=14, return_dict_in_generate=True)
    out = model.generate(input_ids=ids, attention_mask=am, max_length=14, **PROBE)
    assert torch.equal(out.raw_ids, base.raw_ids) and torch.equal(out.sequences, base.sequences)
    assert len(out.encoder_attentions) == 2 and out.encoder_attentions[0].shape == (B, 4, S, S)
    assert len(out.encoder_hidden_states) == 3 and out.encoder_hidden_states[-1].shape == (B, S, cfg.hidden_size)
    assert out.cross_attentions[0][0].shape == (B, cfg.num_attention_heads, 1, S)
    assert (out.cross_attentions[0][0][1, :, :, 5:] == 0).all()   # padded description positions get no weight
