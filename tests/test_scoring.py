"""ParlerTTSForConditionalGeneration.forward(labels=...): teacher-forced scoring (modeling_parler_tts.py:2695-2880, loss :1922-1974).

Host tests pin shift_tokens_right and the label mask against tests/golden/scoring.npz (written by the reference's own code) and the
shim's argument validation.  GPU tests: fp32 against the fixture; the fused bf16 heads + cross-entropy kernel against the unfused
logits at the Mini widths and at the tile edges; the loss against the oracle; scoring a greedy generation's own codes; batch shards.
"""
import os

import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg, tiny_dac_cfg

DEV = "cuda"


def _fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "scoring.npz"))


def _loss64(logits_bktv, labels, dec_bkt, cfg, reduction, weights):
    """The reference's loss in float64 from logits [B*K, T, V] with the shim's mask."""
    from parler_tts_b200.modeling import scoring_label_mask
    B, T, K = labels.shape
    lab, mask = scoring_label_mask(torch.as_tensor(labels), torch.as_tensor(dec_bkt).reshape(B * K, T), cfg.bos_token_id, cfg.eos_token_id)
    lp = torch.log_softmax(torch.as_tensor(logits_bktv, dtype=torch.float64).reshape(B, K, T, -1), dim=-1)
    per = []
    for k in range(K):
        m = mask[..., k]
        nll = -lp[:, k].gather(-1, lab[..., k].clamp(min=0)[..., None])[..., 0][m]
        per.append(nll.mean() if reduction == "mean" else nll.sum())
    per = torch.stack(per)
    loss = (per * torch.tensor(weights, dtype=torch.float64)).sum() / sum(weights) if weights is not None else per.sum() / K
    return float(loss), per.numpy()


# ---- host ------------------------------------------------------------------------------------------------------------------------
def test_shift_and_label_mask_reproduce_reference_fixture(golden_dir):
    from parler_tts_b200.modeling import shift_tokens_right
    z = _fixture(golden_dir)
    cfg = tiny_cfg()
    labels = torch.from_numpy(z["labels"])
    dec = shift_tokens_right(labels, cfg.pad_token_id, cfg.bos_token_id).transpose(1, 2)
    assert np.array_equal(dec.numpy(), z["dec"])
    for red in ("mean", "sum"):
        for wname, w in (("nw", None), ("w", list(z["weights"]))):
            loss, per = _loss64(z["logits"], z["labels"], z["dec"], cfg, red, w)
            np.testing.assert_allclose(per, z[f"{red}_{wname}_per_codebook"], rtol=1e-5)
            assert abs(loss - float(z[f"{red}_{wname}_loss"])) <= 1e-5 * abs(loss)


def test_check_scoring_inputs_validation():
    from parler_tts_b200.modeling import check_scoring_inputs
    B, K, V, T = 2, 4, 96, 6
    kw = dict(batch_size=B, num_codebooks=K, vocab_size=V, pad_token_id=64, decoder_start_token_id=65, prompt_len=3,
              max_position_embeddings=128)
    labels = torch.randint(0, V, (B, T, K))
    labels[1, 4:] = -100
    lab, dec = check_scoring_inputs(labels, None, None, **kw)
    assert dec.shape == (B * K, T) and bool((dec.reshape(B, K, T)[:, :, 0] == 65).all())
    assert torch.equal(check_scoring_inputs(None, dec.reshape(B, K, T), None, **kw)[1], dec)   # [B, K, T] is [B*K, T]
    check_scoring_inputs(labels, None, torch.tensor([[1] * T, [1] * 4 + [0] * 2]), **kw)   # right padding is accepted
    bad_labels = [labels.clone().fill_(V), labels.clone().fill_(-1), labels.float(), labels[:, :, :3], labels[:1]]
    for bl in bad_labels:
        with pytest.raises(ValueError):
            check_scoring_inputs(bl, None, None, **kw)
    for bd in (torch.full((B * K, T), V + 1), torch.full((B * K, T), -1), torch.zeros(B * K + 1, T, dtype=torch.long),
               torch.zeros(B * K, T + 1, dtype=torch.long)):
        with pytest.raises(ValueError):
            check_scoring_inputs(labels, bd, None, **kw)
    check_scoring_inputs(labels, torch.full((B * K, T), V), None, **kw)   # vocab_size itself is an embedding row
    for bm in (torch.tensor([[0] + [1] * (T - 1)] * B), torch.tensor([[1, 0, 1, 1, 1, 1]] * B), torch.ones(B, T + 1), torch.full((B, T), 2)):
        with pytest.raises(ValueError, match="decoder_attention_mask"):
            check_scoring_inputs(labels, None, bm, **kw)
    with pytest.raises(ValueError, match="max_position_embeddings"):
        check_scoring_inputs(labels, None, None, **dict(kw, prompt_len=123))
    with pytest.raises(ValueError, match="labels"):
        check_scoring_inputs(None, None, None, **kw)


def test_forward_rejects_calls_it_cannot_serve():
    from parler_tts_b200 import ParlerTTSForConditionalGeneration
    m = object.__new__(ParlerTTSForConditionalGeneration)   # these checks come before any device work
    with pytest.raises(ValueError, match="does not take"):
        m.forward(labels=torch.zeros(1, 2, 4, dtype=torch.long), past_key_values=None)
    with pytest.raises(ValueError, match="loss_reduction"):
        m.forward(labels=torch.zeros(1, 2, 4, dtype=torch.long), loss_reduction="none")
    with pytest.raises(ValueError, match="decoder_input_ids"):
        m.forward(input_values=torch.zeros(1, 1, 512))


# ---- GPU -------------------------------------------------------------------------------------------------------------------------
def _model(cfg, seed, dtype, head_std=None):
    from oracle.weights import make_dac_weights, make_decoder_weights
    from tests.helpers import build_product_model
    w = make_decoder_weights(cfg, seed=seed, head_std=head_std)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    return w, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=2), dtype=dtype)


@pytest.mark.gpu
def test_fp32_matches_reference_fixture(golden_dir):
    """fp32, tiny shape: logits within 2e-4 and both reductions, with and without codebook_weights, within 1e-5 relative."""
    z = _fixture(golden_dir)
    cfg = tiny_cfg()
    _, model = _model(cfg, seed=13, dtype=torch.float32)
    g = lambda k: torch.from_numpy(z[k]).to(DEV)
    args = dict(encoder_outputs=(g("enc"),), attention_mask=g("enc_mask"), prompt_hidden_states=g("prompt"),
                prompt_attention_mask=g("pmask"), labels=g("labels"))
    for red in ("mean", "sum"):
        for wname, w in (("nw", None), ("w", [float(x) for x in z["weights"]])):
            model.config.decoder.codebook_weights = w
            out = model(**args, loss_reduction=red, return_logits=True)
            assert float(np.abs(out.logits.cpu().numpy() - z["logits"]).max()) < 2e-4
            for o in (out, model(**args, loss_reduction=red)):
                ref = float(z[f"{red}_{wname}_loss"])
                assert abs(float(o.loss) - ref) <= 1e-5 * abs(ref), (red, wname, float(o.loss), ref)
                np.testing.assert_allclose(torch.stack(o.per_codebook_losses).cpu().numpy(), z[f"{red}_{wname}_per_codebook"], rtol=1e-5)
    model.config.decoder.codebook_weights = None


_MINI = {}


def _mini(K=9):
    """bf16 model at the Mini widths (H 1024, V 1088) with 2 layers; logits of a few units (head_std 0.1)."""
    if K not in _MINI:
        cfg = mini_cfg(num_hidden_layers=2, num_codebooks=K, max_position_embeddings=512)
        _MINI[K] = (cfg,) + _model(cfg, seed=31, dtype=torch.bfloat16, head_std=0.1)
    return _MINI[K]


def _inputs(cfg, B, T, P, S, seed):
    from tests.helpers import synth_inputs
    enc, enc_mask, prompt, pmask = synth_inputs(cfg, B, S, P, seed=seed)
    g = torch.Generator().manual_seed(seed)
    labels = torch.randint(0, cfg.vocab_size, (B, T, cfg.num_codebooks), generator=g)
    labels[:, ::7, 0] = cfg.vocab_size - 1
    labels[:, 1::5, -1] = 0
    labels[:, 2::11, :] = -100
    labels[:, 3::13, 0] = cfg.bos_token_id
    return dict(encoder_outputs=(enc.to(DEV),), attention_mask=enc_mask.to(DEV), prompt_hidden_states=None if P == 0 else prompt.to(DEV),
                prompt_attention_mask=None if P == 0 else pmask.to(DEV), labels=labels.to(DEV))


def _nll64(logits, labels, dec, cfg):
    """float64 log-softmax NLL [B, T, K] of logits [B*K, T, V] (0 where the cell is not counted)."""
    from parler_tts_b200.modeling import scoring_label_mask
    B, T, K = labels.shape
    lab, mask = scoring_label_mask(labels.cpu(), dec.cpu(), cfg.bos_token_id, cfg.eos_token_id)
    lp = torch.log_softmax(logits.cpu().double().reshape(B, K, T, -1), dim=-1).permute(0, 2, 1, 3)   # [B, T, K, V]
    nll = -lp.gather(-1, lab.clamp(min=0)[..., None])[..., 0]
    return torch.where(mask, nll, torch.zeros_like(nll)), mask


@pytest.mark.gpu
@pytest.mark.parametrize("K,B,T", [(9, 1, 127), (9, 2, 64), (9, 3, 43), (1, 1, 129), (9, 3, 126), (1, 1, 383)])
def test_bf16_fused_matches_unfused_logits(K, B, T):
    """The fused kernel's token_losses against a float64 log-softmax of the logits the unfused route returns for the same inputs:
    B*T label rows 127, 128, 129, 378 and 383 (partial and whole 128-row tiles), 1 and 9 codebooks, labels at columns 0 and V-1,
    BOS and -100 labels.  The two differ only in the heads' accumulation order, so a logit may move by one bf16 rounding step
    (2^-8 relative); that bounds the tolerance.  Measured on an H100: the largest difference over these cases was 3.1e-2 (K = 9,
    B*T = 129), one rounding step of a logit in [4, 8); the others were 2e-4 .. 9e-3."""
    from parler_tts_b200.modeling import check_scoring_inputs
    cfg, _, model = _mini(K)
    args = _inputs(cfg, B, T, P=8, S=16, seed=B * 1000 + T)
    fused = model(**args)
    full = model(**args, return_logits=True)
    _, dec = check_scoring_inputs(args["labels"].cpu(), None, None, batch_size=B, num_codebooks=K, vocab_size=cfg.vocab_size,
                                  pad_token_id=cfg.pad_token_id, decoder_start_token_id=cfg.bos_token_id, prompt_len=8,
                                  max_position_embeddings=512)
    ref, mask = _nll64(full.logits, args["labels"], dec, cfg)
    got = fused.token_losses.cpu().double()
    assert bool((got[~mask] == 0).all())
    lab_logit = full.logits.cpu().double().reshape(B, K, T, -1).permute(0, 2, 1, 3).abs().amax(-1)
    diff = (got - ref).abs()
    print(f"[score] K={K} B*T={B * T}: fused vs unfused token NLL, largest difference {float(diff.max()):.3e}")
    assert bool((diff <= 2.0 ** -7 * lab_logit.clamp(min=1.0) + 1e-4).all()), float(diff.max())
    # the unfused route's own NLL is the float64 one up to fp32 rounding
    assert float((full.token_losses.cpu().double() - ref).abs().max()) < 1e-4


@pytest.mark.gpu
def test_bf16_zero_tokens_and_masked_utterance():
    """A mean over no counted cell is NaN (as torch's CrossEntropyLoss gives), a sum is 0; an utterance whose labels are all -100
    scores 0 everywhere and leaves the others unchanged."""
    cfg, _, model = _mini(9)
    args = _inputs(cfg, 3, 40, P=0, S=16, seed=5)
    base = model(**args)
    args["labels"][1] = -100
    part = model(**args)
    assert bool((part.token_losses[1] == 0).all())
    assert torch.equal(part.token_losses[0], base.token_losses[0]) and torch.equal(part.token_losses[2], base.token_losses[2])
    args["labels"][:] = -100
    none = model(**args)
    assert bool(torch.isnan(none.loss)) and all(bool(torch.isnan(p)) for p in none.per_codebook_losses)
    assert float(model(**args, loss_reduction="sum").loss) == 0.0


@pytest.mark.gpu
def test_bf16_loss_matches_oracle():
    """The bf16 loss against the oracle's full-prefix logits (oracle/decoder.py), within the oracle's own bf16 noise (its bf16 loss
    against its fp32 loss)."""
    from oracle.decoder import OracleDecoder
    from parler_tts_b200.modeling import check_scoring_inputs
    cfg, w, model = _mini(9)
    B, T, P, S = 2, 48, 8, 16
    args = _inputs(cfg, B, T, P=P, S=S, seed=77)
    labels = args["labels"].cpu()
    _, dec = check_scoring_inputs(labels, None, None, batch_size=B, num_codebooks=9, vocab_size=cfg.vocab_size,
                                  pad_token_id=cfg.pad_token_id, decoder_start_token_id=cfg.bos_token_id, prompt_len=P,
                                  max_position_embeddings=512)
    enc, em = args["encoder_outputs"][0].cpu().float(), args["attention_mask"].cpu()
    pr, pm = args["prompt_hidden_states"].cpu().float(), args["prompt_attention_mask"].cpu()
    ref = {}
    for dt in (torch.float32, torch.bfloat16):
        lo = OracleDecoder(cfg, w, dt).prefill(dec, enc, em, pr, pm)[:, -T:].float()
        ref[dt] = _loss64(lo, labels.numpy(), dec.numpy(), cfg, "mean", None)[0]
    got = float(model(**args).loss)
    noise = abs(ref[torch.bfloat16] - ref[torch.float32])
    print(f"[score] loss {got:.6f}, oracle fp32 {ref[torch.float32]:.6f}, oracle bf16 {ref[torch.bfloat16]:.6f}")
    assert abs(got - ref[torch.float32]) <= 3 * noise + 1e-3


@pytest.mark.gpu
def test_scoring_a_greedy_generation_picks_its_tokens():
    """Score a greedy generate()'s own codes: at every free cell (not a delay-pattern BOS/PAD cell, before the utterance's EOS),
    the scoring logits' argmax is the generated token, except where the top-2 margin is below twice the logit noise (two bf16
    rounding steps of the top logit)."""
    from oracle.delay_pattern import build_delay_pattern_mask
    cfg, _, model = _mini(9)
    B, S, L = 2, 16, 40
    args = _inputs(cfg, B, 4, P=0, S=S, seed=3)
    _, out = model.generate(encoder_outputs=args["encoder_outputs"], attention_mask=args["attention_mask"], do_sample=False,
                            max_length=L, return_codes=True)
    raw = out.raw_ids.cpu()                                 # [B*K, n] delayed, BOS column first
    K, n = cfg.num_codebooks, raw.shape[1]
    dec, labels = raw[:, :-1], raw[:, 1:].reshape(B, K, n - 1).transpose(1, 2).contiguous()
    sc = model(encoder_outputs=args["encoder_outputs"], attention_mask=args["attention_mask"], decoder_input_ids=dec,
               labels=labels.to(DEV), return_logits=True)
    logits = sc.logits.cpu().float()                        # [B*K, n-1, V]: position t predicts column t+1
    _, mask = build_delay_pattern_mask(raw[:, :1].numpy(), cfg.bos_token_id, cfg.pad_token_id, n, K)
    top2 = logits.topk(2, dim=-1).values
    margin, noise = top2[..., 0] - top2[..., 1], 2.0 ** -7 * top2[..., 0].abs()
    checked = close = 0
    for r in range(B * K):
        b = r // K
        eos_cols = (raw[b * K] == cfg.eos_token_id).nonzero()
        end = int(eos_cols[0]) if len(eos_cols) else n   # codebook 0's EOS ends the utterance's free cells
        for c in range(1, min(end, n)):
            tok = int(raw[r, c])
            if mask[r, c] != -1 or tok == cfg.eos_token_id:
                continue
            pick = int(logits[r, c - 1].argmax())
            if pick == cfg.eos_token_id:   # the processor may withhold EOS from a codebook; the draw then is the runner-up
                continue
            checked += 1
            if pick != tok:
                assert float(margin[r, c - 1]) < 2 * float(noise[r, c - 1]), (r, c)
                close += 1
    print(f"[score] greedy tie: {checked} free cells checked, {close} within the noise margin")
    assert checked > 100


@pytest.mark.gpu
def test_batch_above_one_shard_equals_single_utterances():
    """40 utterances run as 32 + 8: token_losses bit-identical to 40 single-utterance calls, loss (mean and sum) within fp32
    summation noise.  P + T and S are >= 128 so a single utterance's prefill takes the same wgmma GEMMs as the batch."""
    from parler_tts_b200.modeling import scoring_label_mask
    cfg, _, model = _mini(9)
    B, T, P, S = 40, 130, 8, 128
    args = _inputs(cfg, B, T, P=P, S=S, seed=40)
    whole = {red: model(**args, loss_reduction=red) for red in ("mean", "sum")}
    one = []
    for b in range(B):
        sl = slice(b, b + 1)
        a1 = dict(encoder_outputs=(args["encoder_outputs"][0][sl],), attention_mask=args["attention_mask"][sl],
                  prompt_hidden_states=args["prompt_hidden_states"][sl], prompt_attention_mask=args["prompt_attention_mask"][sl],
                  labels=args["labels"][sl])
        one.append(model(**a1, loss_reduction="sum").token_losses)
    one = torch.cat(one)
    assert torch.equal(whole["mean"].token_losses, one)
    from parler_tts_b200.modeling import shift_tokens_right
    dec = shift_tokens_right(args["labels"].cpu(), cfg.pad_token_id, cfg.bos_token_id).transpose(1, 2).reshape(B * 9, T)
    _, mask = scoring_label_mask(args["labels"].cpu(), dec, cfg.bos_token_id, cfg.eos_token_id)
    s = one.cpu().double().sum(dim=(0, 1))
    per_mean, per_sum = s / mask.sum(dim=(0, 1)), s
    assert abs(float(whole["mean"].loss) - float(per_mean.mean())) <= 1e-5 * abs(float(per_mean.mean()))
    assert abs(float(whole["sum"].loss) - float(per_sum.mean())) <= 1e-5 * abs(float(per_sum.mean()))
