"""config.prompt_cross_attention: the transcript prompt as cross-attention keys after the description (modeling_parler_tts.py
:2397-2402, :2791-2811, :3099-3130).

Host tests: prompt_cross_states and the oracle's restatement against tests/golden/prompt_cross.npz (written by the reference's own
code) for the four mask combinations, the oracle decoder over those states against the reference's logits, the two rejected
calls and the prompt-length limit, and the position table in the broadcast list.  GPU tests: fp32 generate() and
forward(labels=...) against the oracle and the fixture; bf16 Mini on the cluster step kernel at S + P = 96, 66 and 512 keys,
bit-identical to step.cu and within the bf16 noise of the oracle; generate() with the prompt bit-identical to generate() over the
assembled states (shards, streamer, continuation); the probes' shapes; a world-size-2 weight broadcast.
"""
import os
import types

import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg

DEV = "cuda"


def _fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "prompt_cross.npz"))


def _case_inputs(z, ci):
    use_em, use_pm = (bool(x) for x in z["cases"][ci])
    enc_mask = torch.from_numpy(z["enc_mask"]) if use_em else None
    pmask = torch.from_numpy(z["pmask"]) if use_pm else None
    return torch.from_numpy(z["enc"]), enc_mask, torch.from_numpy(z["prompt_ids"]), pmask


def _golden_mask(z, ci):
    return torch.from_numpy(z[f"c{ci}_mask"]) if int(z[f"c{ci}_has_mask"]) else None


# ---- host ----------------------------------------------------------------------------------------------------------------------
def test_assembly_matches_reference_fixture(golden_dir):
    """prompt_cross_states (the library's assembly, on CPU tensors) and the oracle's restatement give the reference's states and
    mask bit for bit in fp32, for every combination of description and prompt mask."""
    from oracle.weights import make_decoder_weights
    from parler_tts_b200.modeling import _sinusoidal_table, prompt_cross_states
    from tests.prompt_cross_oracle import assemble
    z = _fixture(golden_dir)
    cfg = tiny_cfg()
    w = make_decoder_weights(cfg, seed=13)
    table = _sinusoidal_table(cfg.max_position_embeddings, cfg.hidden_size)
    for ci in range(len(z["cases"])):
        enc, em, ids, pm = _case_inputs(z, ci)
        want_states, want_mask = torch.from_numpy(z[f"c{ci}_states"]), _golden_mask(z, ci)
        for states, mask in (prompt_cross_states(enc, em, ids, pm, w["embed_prompts.weight"], table),
                             assemble(enc, em, ids, pm, w["embed_prompts.weight"], cfg.max_position_embeddings)):
            assert torch.equal(states, want_states), ci
            assert (mask is None) == (want_mask is None), ci
            if mask is not None:
                assert torch.equal(mask, want_mask), ci


def test_oracle_decoder_over_assembled_states_matches_reference_logits(golden_dir):
    """OracleDecoder over the assembled keys with no prompt prefix reproduces the reference's ParlerTTSForCausalLM logits."""
    from oracle.decoder import OracleDecoder
    from oracle.weights import make_decoder_weights
    z = _fixture(golden_dir)
    cfg = tiny_cfg()
    dec = OracleDecoder(cfg, make_decoder_weights(cfg, seed=13), torch.float32)
    B, K, T, P, S = (int(x) for x in z["meta"])
    ids = torch.from_numpy(z["dec"]).reshape(B * K, T)
    for ci in range(len(z["cases"])):
        lo = dec.prefill(ids, torch.from_numpy(z[f"c{ci}_states"]), _golden_mask(z, ci), None, None)
        assert float((lo - torch.from_numpy(z[f"c{ci}_logits"])).abs().max()) < 1e-4, ci


def _cpu_model(cross=True):
    """A model object with only the attributes the argument checks read (they come before any device work)."""
    from parler_tts_b200 import GenerationConfig, ParlerTTSForConditionalGeneration
    m = object.__new__(ParlerTTSForConditionalGeneration)
    m.prompt_cross_attention = cross
    m.generation_config = GenerationConfig(max_length=20, do_sample=False)
    return m


def test_incoherent_calls_are_rejected_before_device_work():
    m = _cpu_model()
    enc = (torch.zeros(1, 3, 8),)
    with pytest.raises(ValueError, match="prompt_input_ids"):
        m.generate(encoder_outputs=enc, prompt_hidden_states=torch.zeros(1, 2, 8))
    labels = torch.zeros(1, 2, 4, dtype=torch.long)
    with pytest.raises(ValueError, match="encoder_outputs"):
        m.forward(encoder_outputs=enc, prompt_input_ids=torch.zeros(1, 2, dtype=torch.long), labels=labels)
    with pytest.raises(ValueError, match="encoder_outputs"):
        m.forward(encoder_outputs=enc, prompt_hidden_states=torch.zeros(1, 2, 8), labels=labels)


def test_prompt_longer_than_the_position_table_is_rejected():
    from parler_tts_b200.modeling import _sinusoidal_table, prompt_cross_states
    table = _sinusoidal_table(16, 8)
    emb = torch.zeros(100, 8)
    states, mask = prompt_cross_states(torch.zeros(2, 3, 8), None, torch.zeros(2, 16, dtype=torch.long), None, emb, table)
    assert states.shape == (2, 19, 8) and mask is None
    with pytest.raises(ValueError, match="max_position_embeddings"):
        prompt_cross_states(torch.zeros(2, 3, 8), None, torch.zeros(2, 17, dtype=torch.long), None, emb, table)
    with pytest.raises(ValueError, match="prompt must be"):
        prompt_cross_states(torch.zeros(2, 3, 8), None, torch.zeros(3, 4, dtype=torch.long), None, emb, table)


def test_position_table_is_in_the_broadcast_list():
    from parler_tts_b200.dist import model_weight_tensors
    fill = lambda *s: torch.zeros(*s)
    base = dict(decoder=types.SimpleNamespace(engine=types.SimpleNamespace(blob=fill(4))), audio_encoder=types.SimpleNamespace(blob=fill(4)),
                embed_prompts_weight=fill(3, 2), enc_to_dec_proj=None)
    table = fill(5, 2)
    assert not any(t is table for t in model_weight_tensors(types.SimpleNamespace(**base, embed_positions_weight=None)))
    assert any(t is table for t in model_weight_tensors(types.SimpleNamespace(**base, embed_positions_weight=table)))


# ---- GPU -----------------------------------------------------------------------------------------------------------------------
class _FixedEncoder(torch.nn.Module):
    """Stands in for the T5 encoder: returns the given description states (already multiplied by their mask), cut to the ids'
    shape, so forward() runs its text-encoder branch."""

    def __init__(self, states):
        super().__init__()
        self.states = torch.nn.Parameter(states, requires_grad=False)

    def forward(self, input_ids=None, attention_mask=None, return_dict=True, **kw):
        return types.SimpleNamespace(last_hidden_state=self.states[:input_ids.shape[0], :input_ids.shape[1]].clone())


def _cross_model(cfg, w, dtype, text_encoder=None):
    from oracle.weights import make_dac_weights
    from parler_tts_b200 import ParlerTTSConfig, ParlerTTSForConditionalGeneration
    from tests.helpers import product_dac_config, product_decoder_config
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    pc = ParlerTTSConfig(vocab_size=cfg.text_vocab_size, text_encoder={}, audio_encoder=product_dac_config(dcfg),
                         decoder=product_decoder_config(cfg), prompt_cross_attention=True)
    m = ParlerTTSForConditionalGeneration(pc, device=DEV, dtype=dtype, text_encoder=text_encoder)
    m.load_state_dict(w, dac_state_dict=make_dac_weights(dcfg, seed=2))
    return m


@pytest.mark.gpu
def test_fp32_generate_matches_oracle(golden_dir):
    """fp32, tiny shape, the fixture's inputs in all four mask combinations: greedy tokens bit-exact against the oracle over the
    assembled keys, every step's logits within 2e-4, and the decoder attentions without prompt rows."""
    from oracle.decoder import OracleDecoder
    from oracle.delay_pattern import apply_delay_pattern_mask
    from oracle.sampling import generate_tokens
    from oracle.weights import make_decoder_weights
    from tests.prompt_cross_oracle import assemble
    z = _fixture(golden_dir)
    cfg = tiny_cfg()
    w = make_decoder_weights(cfg, seed=13, head_std=0.5)   # logits of a few units: greedy margins far above fp32 noise
    model = _cross_model(cfg, w, torch.float32)
    L = 24
    for ci in range(len(z["cases"])):
        enc, em, ids, pm = _case_inputs(z, ci)
        states, mask = assemble(enc, em, ids, pm, w["embed_prompts.weight"], cfg.max_position_embeddings)
        ref = generate_tokens(OracleDecoder(cfg, w, torch.float32), cfg, states, mask, None, None, dict(max_length=L, do_sample=False),
                              collect_logits=True)
        cuda = lambda t: None if t is None else t.to(DEV)
        out = model.generate(encoder_outputs=(enc.to(DEV),), attention_mask=cuda(em), prompt_input_ids=ids.to(DEV),
                             prompt_attention_mask=cuda(pm), do_sample=False, max_length=L, return_dict_in_generate=True,
                             output_logits=True)
        want = apply_delay_pattern_mask(ref["raw_ids"], ref["delay_mask"])
        assert np.array_equal(out.raw_ids.cpu().numpy(), want), ci
        assert len(out.logits) == len(ref["logits"])
        err = max(float(np.abs(a.cpu().numpy() - b).max()) for a, b in zip(out.logits, ref["logits"]))
        assert err < 2e-4, (ci, err)


@pytest.mark.gpu
def test_fp32_forward_labels_matches_reference_fixture(golden_dir):
    """forward(input_ids=..., prompt_input_ids=..., labels=...) through the text-encoder branch: logits within 2e-4 of the
    reference's, the loss within 1e-5 relative, token_losses within 2e-4 of a float64 NLL of the reference's logits; the same with
    the prompt passed as prompt_hidden_states (the embedded ids)."""
    from oracle.weights import make_decoder_weights
    from parler_tts_b200.modeling import scoring_label_mask
    z = _fixture(golden_dir)
    cfg = tiny_cfg()
    w = make_decoder_weights(cfg, seed=13)
    B, K, T, P, S = (int(x) for x in z["meta"])
    enc = torch.from_numpy(z["enc"])
    model = _cross_model(cfg, w, torch.float32, text_encoder=_FixedEncoder(enc.to(DEV)))
    labels = torch.from_numpy(z["labels"])
    lab, cnt = scoring_label_mask(labels, torch.from_numpy(z["dec"]).reshape(B * K, T), cfg.bos_token_id, cfg.eos_token_id)
    desc_ids = torch.zeros(B, S, dtype=torch.long, device=DEV)
    for ci in range(len(z["cases"])):
        _, em, ids, pm = _case_inputs(z, ci)
        cuda = lambda t: None if t is None else t.to(DEV)
        ref_logits = torch.from_numpy(z[f"c{ci}_logits"])
        lp = torch.log_softmax(ref_logits.double().reshape(B, K, T, -1), -1).permute(0, 2, 1, 3)
        nll = -lp.gather(-1, lab.clamp(min=0)[..., None])[..., 0]
        ref_tok = torch.where(cnt, nll, torch.zeros_like(nll))
        prompts = dict(prompt_input_ids=ids.to(DEV)), dict(prompt_hidden_states=w["embed_prompts.weight"][ids].to(DEV))
        for prompt in prompts:
            out = model(input_ids=desc_ids, attention_mask=cuda(em), prompt_attention_mask=cuda(pm), labels=labels.to(DEV),
                        return_logits=True, **prompt)
            assert float((out.logits.cpu() - ref_logits).abs().max()) < 2e-4, ci
            ref_loss = float(z[f"c{ci}_loss"])
            assert abs(float(out.loss) - ref_loss) <= 1e-5 * abs(ref_loss), (ci, float(out.loss), ref_loss)
            assert float((out.token_losses.cpu().double() - ref_tok).abs().max()) < 2e-4, ci


_MINI = {}


def _mini():
    """bf16 model at the Mini widths (H 1024, V 1088, 9 codebooks) with 2 layers."""
    if "m" not in _MINI:
        from oracle.weights import make_decoder_weights
        cfg = mini_cfg(num_hidden_layers=2, max_position_embeddings=512)
        w = make_decoder_weights(cfg, seed=91, head_std=0.2)
        _MINI["m"] = (cfg, w, _cross_model(cfg, w, torch.bfloat16))
    return _MINI["m"]


def _mini_inputs(cfg, B, S, P, seed):
    from tests.helpers import synth_inputs
    enc, em, _, pm = synth_inputs(cfg, B, S, P, seed=seed)
    ids = torch.randint(0, cfg.text_vocab_size, (B, P), generator=torch.Generator().manual_seed(seed + 1))
    return enc.bfloat16().float(), em, ids, pm


def _need_132_sm_class_device():
    props = torch.cuda.get_device_properties(0)
    if props.multi_processor_count < 128:
        pytest.skip(f"{props.name} has {props.multi_processor_count} SMs: fewer than the 64 co-resident clusters of 2 Mini needs")


@pytest.mark.gpu
@pytest.mark.parametrize("S,P", [(64, 32), (37, 29), (64, 448)])
def test_bf16_mini_cluster_kernel(monkeypatch, S, P):
    """Mini widths, bf16, B = 32 at S + P = 96 (the benchmark's S and P), 66 (not a multiple of 32) and 512 cross keys.
    generate() decodes on the cluster step kernel; teacher-forced on the bf16 oracle's greedy history, the cluster kernel's logits
    equal step.cu's bit for bit at every step and stay within the bf16 noise bound of test_gpu_parity_bench_config (3 % of the
    largest logit)."""
    from oracle.decoder import OracleDecoder
    from oracle.sampling import generate_tokens
    from parler_tts_b200.modeling import GenSession
    from tests.prompt_cross_oracle import assemble
    _need_132_sm_class_device()
    monkeypatch.delenv("PTTS_STEP", raising=False)
    cfg, w, model = _mini()
    B, steps = 32, 24
    L = steps + 1
    enc, em, ids, pm = _mini_inputs(cfg, B, S, P, seed=S * 1000 + P)
    model.generate(encoder_outputs=(enc.to(DEV),), attention_mask=em.to(DEV), prompt_input_ids=ids.to(DEV),
                   prompt_attention_mask=pm.to(DEV), do_sample=False, max_length=8)
    assert model.decoder.engine._sessions[(B, 0, S + P)].fused == 2, "generate() does not decode on the cluster step kernel"

    states, mask = assemble(enc, em, ids, pm, w["embed_prompts.weight"], cfg.max_position_embeddings, torch.bfloat16)
    ref = generate_tokens(OracleDecoder(cfg, w, torch.bfloat16), cfg, states.float(), mask, None, None,
                          dict(max_length=L, do_sample=False), collect_logits=True)
    n = min(steps, ref["raw_ids"].shape[1] - 1)
    got = {}
    for mode, kind in (("legacy", 1), ("cluster", 2)):
        monkeypatch.setenv("PTTS_STEP", mode)
        sess = GenSession(model.decoder.engine, B, 0, S + P, L)
        try:
            sess.begin(L, do_sample=False)
            sess.prefill(None, None, states.to(DEV), mask)
            assert sess.fused == kind, (mode, sess.fused)
            logits = []
            for t in range(n):
                if t > 0:
                    sess.decode_forward()
                logits.append(sess.logits.cpu().numpy().copy())
                sess.sample(forced=torch.from_numpy(ref["raw_ids"][:, t + 1].copy()))
            torch.cuda.synchronize()
            got[mode] = np.stack(logits)
        finally:
            sess.close()
    assert np.array_equal(got["cluster"].view(np.uint32), got["legacy"].view(np.uint32)), "step2.cu and step.cu differ"
    rel = max(float(np.abs(a - b).max()) / float(np.abs(b).max()) for a, b in zip(got["cluster"], ref["logits"][:n]))
    print(f"\n[prompt-cross] S={S} P={P}: max |logit err| / max|logit| = {rel:.4f} over {n} steps")
    assert rel < 0.03, rel


class _Collect:
    def __init__(self):
        self.cols = []

    def put(self, v):
        self.cols.append(v.reshape(v.shape[0], -1).clone())

    def end(self):
        pass


@pytest.mark.gpu
def test_prompt_equals_generate_over_the_assembled_states():
    """generate(prompt_input_ids=p, attention_mask=m, prompt_attention_mask=pm) gives the codes and audio of
    generate(encoder_outputs=(assembled,), attention_mask=assembled mask) bit for bit: sampled, at B = 40 (shards of 32), with a
    streamer (the same streamed columns) and continuing from decoder_input_ids."""
    from parler_tts_b200.modeling import prompt_cross_states
    cfg, w, model = _mini()
    K = cfg.num_codebooks
    gen = dict(do_sample=True, temperature=0.9, top_k=50, seed=11, max_length=28, return_codes=True)
    for B, extra in ((40, {}), (3, "streamer"), (4, "continue")):
        enc, em, ids, pm = (t.to(DEV) for t in _mini_inputs(cfg, B, 16, 12, seed=B))
        states, mask = prompt_cross_states(enc.bfloat16(), em, ids, pm, model.embed_prompts_weight, model.embed_positions_weight)
        assert states.shape == (B, 28, cfg.hidden_size) and mask.shape == (B, 28)
        kw = dict(gen)
        if extra == "continue":
            kw["decoder_input_ids"] = torch.randint(0, cfg.codebook_size, (B * K, 5), generator=torch.Generator().manual_seed(3)).to(DEV)
        runs = []
        for call in (dict(encoder_outputs=(enc,), attention_mask=em, prompt_input_ids=ids, prompt_attention_mask=pm),
                     dict(encoder_outputs=(states,), attention_mask=mask)):
            streamer = _Collect() if extra == "streamer" else None
            audio, out = model.generate(**call, **kw, streamer=streamer)
            runs.append((audio, out.audio_codes, out.raw_ids, None if streamer is None else torch.cat(streamer.cols, dim=1)))
        (a0, c0, r0, s0), (a1, c1, r1, s1) = runs
        assert torch.equal(c0, c1) and torch.equal(r0, r1) and torch.equal(a0, a1), (B, extra)
        if s0 is not None:
            assert torch.equal(s0, s1)


@pytest.mark.gpu
def test_probes_have_the_prompt_among_the_cross_keys():
    """output_attentions in cross mode: cross_attentions[t][l] is [B, heads, q, S + P] and each row sums to 1 over its unmasked
    keys (masked keys 0); decoder_attentions have no prompt rows (entry 0: q = 1); scores still have one entry per step."""
    from oracle.weights import make_decoder_weights
    cfg = tiny_cfg()
    w = make_decoder_weights(cfg, seed=13)
    model = _cross_model(cfg, w, torch.float32)
    B, S, P, L = 2, 7, 5, 12
    from tests.helpers import synth_inputs
    enc, em, _, pm = synth_inputs(cfg, B, S, P, seed=8)
    ids = torch.randint(0, cfg.text_vocab_size, (B, P), generator=torch.Generator().manual_seed(8))
    out = model.generate(encoder_outputs=(enc.to(DEV),), attention_mask=em.to(DEV), prompt_input_ids=ids.to(DEV),
                         prompt_attention_mask=pm.to(DEV), do_sample=False, max_length=L, return_dict_in_generate=True,
                         output_attentions=True, output_scores=True)
    n = out.raw_ids.shape[1] - 1
    assert len(out.scores) == len(out.cross_attentions) == len(out.decoder_attentions) == n
    keep = torch.cat([em, pm], dim=1).to(DEV).bool()[:, None, None, :]
    for t in range(n):
        q = 1
        assert all(a.shape == (B, cfg.num_attention_heads, q, 1 + t) for a in out.decoder_attentions[t])
        for a in out.cross_attentions[t]:
            assert a.shape == (B, cfg.num_attention_heads, q, S + P)
            assert bool((a.masked_fill(keep, 0) == 0).all())
            assert float((a.masked_fill(~keep, 0).sum(-1) - 1).abs().max()) < 1e-5


def _dist_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle.weights import make_decoder_weights
    from parler_tts_b200.dist import broadcast_model_weights, model_weight_tensors
    cfg = tiny_cfg()
    model = _cross_model(cfg, make_decoder_weights(cfg, seed=13), torch.float32) if rank == 0 else None
    if rank == 0:
        # a checkpoint's own table (here: the sinusoidal one scaled), so that its arrival is visible on rank 1
        model.load_state_dict({**make_decoder_weights(cfg, seed=13), "embed_positions.weights": 2 * model.embed_positions_weight.cpu()})
    else:
        from parler_tts_b200 import ParlerTTSConfig, ParlerTTSForConditionalGeneration
        from tests.helpers import product_dac_config, product_decoder_config
        dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
        model = ParlerTTSForConditionalGeneration(
            ParlerTTSConfig(vocab_size=cfg.text_vocab_size, text_encoder={}, audio_encoder=product_dac_config(dcfg),
                            decoder=product_decoder_config(cfg), prompt_cross_attention=True), device=DEV, dtype=torch.float32)
    listed = any(t is model.embed_positions_weight for t in model_weight_tensors(model))
    broadcast_model_weights(model)
    from parler_tts_b200.modeling import _sinusoidal_table
    arrived = torch.equal(model.embed_positions_weight.cpu(), 2 * _sinusoidal_table(cfg.max_position_embeddings, cfg.hidden_size))
    q.put((rank, listed, arrived, model._side_loaded))
    dist.destroy_process_group()


@pytest.mark.gpu
def test_world_size_2_broadcasts_the_position_table():
    """Two gloo ranks in cross mode: rank 0 loads a checkpoint with its own embed_positions.weights, rank 1 only constructs the
    model; after broadcast_model_weights rank 1 holds rank 0's table."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 500) % 1000
    ps = [ctx.Process(target=_dist_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = sorted(q.get(timeout=300) for _ in ps)
    for p in ps:
        p.join(timeout=60)
    assert res == [(0, True, True, True), (1, True, True, True)], res
