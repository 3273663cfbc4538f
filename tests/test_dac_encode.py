"""DACModel.encode (dac_wrapper/modeling_dac.py:33-104) and generate(input_values=...) (modeling_parler_tts.py:3136-3194).

Host tests pin the CPU oracle to tests/golden/dac_encode.npz (written by transformers' DacModel.encode), the two checkpoint key
layouts and the shim's input validation.  GPU tests run the encode kernels: the generic path against the fixture, the wgmma path
at the 44.1 kHz shape against torch's own bf16 error, the quantizer's choices against an fp64 re-trace, and generate() from a
waveform against generate() from that waveform's codes.
"""
from __future__ import annotations
import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle.config import dac_cfg, tiny_cfg
from oracle.weights import make_dac_weights, make_decoder_weights
from tests.dac_encode_oracle import OracleDACEncoder, make_dac_encoder_weights
from tests.golden.make_dac_encode_golden import encode_cfg, weights
from tests.helpers import product_decoder_config, rms

DEV = "cuda"


def product_codec_config(dcfg):
    from parler_tts_b200 import DACConfig
    return DACConfig(num_codebooks=dcfg.n_codebooks, codebook_size=dcfg.codebook_size, latent_dim=dcfg.hidden_size,
                     codebook_dim=dcfg.codebook_dim, decoder_dim=dcfg.decoder_hidden_size, decoder_rates=tuple(dcfg.upsampling_ratios),
                     encoder_dim=dcfg.get("encoder_hidden_size", 64), encoder_rates=tuple(dcfg.get("downsampling_ratios", [2, 4, 8, 8])))


def _report(name, data):
    """Numbers a GPU test measured: printed, and written as JSON under $PTTS_TEST_REPORT_DIR when that is set."""
    print(name, json.dumps(data))
    out = os.environ.get("PTTS_TEST_REPORT_DIR")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, name + ".json"), "w") as f:
            json.dump(data, f, indent=1)


# ---- host ------------------------------------------------------------------------------------------
def test_oracle_encode_reproduces_fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "dac_encode.npz"))
    cfg = encode_cfg()
    o = OracleDACEncoder(cfg, weights(cfg), torch.float64)
    wav = torch.from_numpy(z["waveform"])
    assert wav.shape[-1] % 512 != 0
    codes = o.encode(wav)
    assert codes.shape == (1,) + z["codes"].shape
    assert np.array_equal(codes[0].numpy(), z["codes"])
    lat = OracleDACEncoder(cfg, weights(cfg)).encoder(torch.from_numpy(z["padded"])).numpy()   # fp32, like the fixture's tolerance
    assert np.abs(lat - z["latents"]).max() <= 1e-5 * np.abs(z["latents"]).max()


def test_frame_count_is_ceil_samples_over_hop():
    cfg = encode_cfg()
    o = OracleDACEncoder(cfg, weights(cfg))
    for n in (1, 511, 512, 513, 1500):
        assert o.encode(torch.zeros(1, 1, n)).shape[-1] == math.ceil(n / 512), n


def _to_descript(sd: dict, n_blocks: int) -> dict:
    """transformers-style encoder / quantizer keys -> descript-audio-codec keys, conv weights as weight-norm (g, v) pairs."""
    out = {}

    def put(key, v):
        if key.endswith(".weight") and v.dim() == 3 and "codebook" not in key:
            g = v.flatten(1).norm(dim=1).view(-1, 1, 1)
            out[key[:-len("weight")] + "weight_g"] = g
            out[key[:-len("weight")] + "weight_v"] = v * 1.7
        else:
            out[key] = v
    unit = {"snake1.": "0.", "conv1.": "1.", "snake2.": "2.", "conv2.": "3."}
    for k, v in sd.items():
        if k.startswith("decoder."):
            continue
        if k.startswith("quantizer."):
            put(k, v)
        elif k.startswith("encoder.conv1."):
            put("encoder.block.0." + k[len("encoder.conv1."):], v)
        elif k.startswith("encoder.snake1."):
            put(f"encoder.block.{n_blocks + 1}." + k[len("encoder.snake1."):], v)
        elif k.startswith("encoder.conv2."):
            put(f"encoder.block.{n_blocks + 2}." + k[len("encoder.conv2."):], v)
        else:
            _, _, bi, rest = k.split(".", 3)
            p = f"encoder.block.{int(bi) + 1}.block."
            if rest.startswith("res_unit"):
                r, tail = rest[len("res_unit")], rest[len("res_unitN."):]
                name = next(n for n in unit if tail.startswith(n))
                put(p + f"{int(r) - 1}.block." + unit[name] + tail[len(name):], v)
            elif rest.startswith("snake1."):
                put(p + "3." + rest[len("snake1."):], v)
            else:
                put(p + "4." + rest[len("conv1."):], v)
    return out


def test_descript_and_transformers_encoder_keys_map_to_the_same_table():
    from parler_tts_b200.dac_wrapper import _dac_encoder_tensor_list, _encoder_state_dict, _fold_weight_norm
    cfg = encode_cfg()
    w = weights(cfg)
    n = len(cfg.downsampling_ratios)
    names = _dac_encoder_tensor_list(product_codec_config(cfg))
    a = _encoder_state_dict(_fold_weight_norm(dict(w)), n)
    d = _to_descript(w, n)
    assert any(k.startswith("encoder.block.1.block.0.block.") for k in d)
    b = _encoder_state_dict(_fold_weight_norm(d), n)
    assert set(names) <= set(a) and set(names) <= set(b)
    for k in names:
        assert a[k].shape == b[k].shape and torch.allclose(a[k], b[k], rtol=1e-5, atol=1e-6), k


def test_encoder_tensor_table_matches_the_library():
    from parler_tts_b200 import DACConfig, _lib
    from parler_tts_b200.dac_wrapper import DACModel, _dac_encoder_tensor_list
    for cfg in (product_codec_config(encode_cfg()), DACConfig()):
        m = DACModel(cfg, device="cpu")
        n = ctypes.c_int32()
        _lib.check(_lib.lib().ptts_dac_encoder_num_tensors(ctypes.byref(m._c), ctypes.byref(n)))
        assert n.value == len(_dac_encoder_tensor_list(cfg))
        assert m.encoder_blob is not None and m.encoder_blob.numel() > 0


def test_encode_input_validation():
    from parler_tts_b200 import DACConfig
    from parler_tts_b200.dac_wrapper import DACModel
    cfg = product_codec_config(encode_cfg())
    m = DACModel(cfg, device="cpu")   # nothing loaded: validation comes first, then the missing encoder
    wav = torch.zeros(2, 1, 1000)
    with pytest.raises(ValueError):
        m.encode(torch.zeros(2, 2, 1000))                          # stereo: the encoder's first conv takes one channel
    with pytest.raises(ValueError):
        m.encode(torch.zeros(2, 3, 1000))
    with pytest.raises(ValueError):
        m.encode(wav, sample_rate=16000)
    with pytest.raises(ValueError):
        m.encode(torch.zeros(2, 1, 0))
    with pytest.raises(ValueError):
        m.encode(torch.zeros(0, 1, 1000))
    for nq in (0, cfg.num_codebooks + 1):
        with pytest.raises(ValueError):
            m.encode(wav, n_quantizers=nq)
    with pytest.raises(RuntimeError, match="encoder weights"):
        m.encode(wav, sample_rate=44100)
    # a codec whose encoder hop differs from the decoder's decodes, but cannot encode
    odd = DACModel(DACConfig(decoder_rates=(8, 8, 4)), device="cpu")
    assert odd.encoder_blob is None
    with pytest.raises(ValueError, match="hop"):
        odd.encode(wav)
    off = DACModel(DACConfig(encoder_dim=0), device="cpu")
    with pytest.raises(ValueError, match="no encoder"):
        off.encode(wav)


def test_encoder_refused_where_the_quantizer_cannot_run():
    """A codebook_dim or latent_dim the quantizer kernel does not take leaves the codec decode-only: no encoder blob, and encode()
    raises before any launch."""
    from parler_tts_b200 import DACConfig
    from parler_tts_b200.dac_wrapper import DACModel
    wav = torch.zeros(1, 1, 1000)
    for kw in (dict(codebook_dim=12), dict(latent_dim=2048)):
        m = DACModel(DACConfig(**kw), device="cpu")
        assert m.encoder_blob is None and m.blob.numel() > 0, kw
        with pytest.raises(ValueError, match="quantizer"):
            m.encode(wav)
    for D in (4, 8, 16):
        assert DACModel(DACConfig(codebook_dim=D, latent_dim=1536), device="cpu").encoder_blob is not None


# ---- GPU -------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_encode_tiny_generic_path_vs_fixture(golden_dir, dtype):
    from parler_tts_b200 import DACModel
    z = np.load(os.path.join(golden_dir, "dac_encode.npz"))
    cfg = encode_cfg()
    w = weights(cfg)
    m = DACModel(product_codec_config(cfg), DEV, dtype).load_state_dict(w)
    wav = torch.from_numpy(z["waveform"])
    B, K, T = z["codes"].shape
    codes, lat = m._encode(wav[:, 0].to(DEV), K, return_latents=True)
    ref = z["latents"].transpose(0, 2, 1)
    got = lat.float().cpu().numpy()
    if dtype == torch.float32:
        assert np.abs(got - ref).max() <= 2e-4 * np.abs(ref).max(), np.abs(got - ref).max()
        near_tie = z["margins"].transpose(1, 0, 2) < 1e-5
        assert np.all((codes.cpu().numpy() == z["codes"]) | near_tie)
    else:   # bf16 storage: as accurate as torch's own bf16 run of the same network on the CPU
        cpu = OracleDACEncoder(cfg, w, torch.bfloat16).encoder(torch.from_numpy(z["padded"]).bfloat16()).float().numpy().transpose(0, 2, 1)
        assert rms(got - ref) <= 1.5 * rms(cpu - ref) + 1e-4, (rms(got - ref), rms(cpu - ref))
    out = m.encode(wav.to(DEV), sample_rate=44100)
    assert out.audio_codes.shape == (1, B, K, T) and out.audio_scales == [None]
    assert torch.equal(out.audio_codes[0], codes) and torch.equal(out[0], out.audio_codes)
    assert torch.equal(m.encode(wav.to(DEV), return_dict=False)[0], out.audio_codes)
    assert torch.equal(m.encode(wav.to(DEV), n_quantizers=2).audio_codes[0], codes[:, :2])
    assert torch.equal(m.encode(wav.to(dtype).to(DEV)).audio_codes[0], codes)   # model-dtype audio: the same rounding


def _real_shape_model(seed_dec=3, seed_enc=7):
    from parler_tts_b200 import DACModel
    dcfg = dac_cfg()
    w = make_dac_weights(dcfg, seed=seed_dec)
    w.update(make_dac_encoder_weights(dcfg, seed=seed_enc))
    return dcfg, w, DACModel(product_codec_config(dcfg), DEV, torch.bfloat16).load_state_dict(w)


def _kernel_path_similarities(z_btz: torch.Tensor, w: dict, K: int, codes: torch.Tensor) -> list:
    """The quantizer's arithmetic as the bf16 kernel does it (bf16 roundings where torch's bf16 ops round, fp32 cosine), in torch
    on the CPU, along the kernel's codes: per codebook the [B, T, codebook_size] similarities it compared."""
    bf = lambda t: t.to(torch.bfloat16).float()
    r, sims = z_btz.float(), []
    for k in range(K):
        q = f"quantizer.quantizers.{k}."
        e = bf(r @ bf(w[q + "in_proj.weight"][:, :, 0]).t() + bf(w[q + "in_proj.bias"]))
        cb = bf(w[q + "codebook.weight"])
        en = e / e.norm(dim=-1, keepdim=True).clamp_min(1e-12)
        sims.append(en @ (cb / cb.norm(dim=1, keepdim=True).clamp_min(1e-12)).t())
        st = bf(e + bf(cb[codes[:, k]] - e))
        r = bf(r - bf(st @ bf(w[q + "out_proj.weight"][:, :, 0]).t() + bf(w[q + "out_proj.bias"])))
    return sims


@pytest.mark.gpu
def test_encode_bf16_real_shape_wgmma_and_quantizer_choices():
    """44.1 kHz shape, B = 2, 44100 + 300 samples, wgmma path.  Latents: RMS error vs the fp32 oracle within 1.5x torch's own
    bf16 CPU error + 1e-4.  Codes: every kernel choice is the fp64 argmax along the kernel's own path, or a near tie whose gap
    is below twice the largest |kernel - fp64| similarity error of this run."""
    dcfg, w, m = _real_shape_model()
    g = torch.Generator().manual_seed(21)
    n = 44100 + 300
    t = torch.arange(n) / 44100.0
    wav = (0.3 * torch.sin(2 * math.pi * 180.0 * t) + 0.1 * torch.randn(2, n, generator=g))[:, None, :]
    K = dcfg.n_codebooks
    codes, lat = m._encode(wav[:, 0].to(DEV), K, return_latents=True)
    T = math.ceil(n / 512)
    assert codes.shape == (2, K, T) and lat.shape == (2, T, dcfg.hidden_size)
    padded = torch.nn.functional.pad(wav, (0, T * 512 - n))
    ref = OracleDACEncoder(dcfg, w).encoder(padded).numpy().transpose(0, 2, 1)
    cpu = OracleDACEncoder(dcfg, w, torch.bfloat16).encoder(padded.bfloat16()).float().numpy().transpose(0, 2, 1)
    got = lat.float().cpu().numpy()
    e_gpu, e_cpu = rms(got - ref), rms(cpu - ref)
    assert rms(ref) > 1e-2
    assert e_gpu <= 1.5 * e_cpu + 1e-4, (e_gpu, e_cpu)

    kc = codes.cpu()
    z64 = lat.cpu().double().permute(0, 2, 1)
    _, sims64 = OracleDACEncoder(dcfg, w, torch.float64).quantize(z64, K, follow=kc)
    sims32 = _kernel_path_similarities(lat.cpu(), w, K, kc)
    err = max(float((a.double() - b).abs().max()) for a, b in zip(sims32, sims64))
    flips, worst, bad = 0, 0.0, []
    for k in range(K):
        s = sims64[k]
        gap = s.max(-1).values - s.gather(-1, kc[:, k, :, None])[..., 0]
        flip = gap > 0
        flips += int(flip.sum())
        if flip.any():
            worst = max(worst, float(gap[flip].max()))
        if bool((gap >= 2 * err).any()):
            bad.append(k)
    _report("dac_encode_quantizer", {"frames": 2 * T, "codebooks": K, "flips": flips, "worst_flip_gap": worst,
                                     "max_similarity_error": err, "latent_rms_err_gpu": e_gpu, "latent_rms_err_torch_bf16": e_cpu})
    assert not bad, (bad, err, worst)


@pytest.mark.gpu
def test_encode_wgmma_vs_generic_path(monkeypatch):
    """B = 32, 2 s: the wgmma path against the generic conv kernel (PTTS_DAC_TC=0) on the same bf16 weights."""
    dcfg, w, m = _real_shape_model()
    g = torch.Generator().manual_seed(5)
    wav = (0.2 * torch.randn(32, 1, 2 * 44100, generator=g)).to(DEV)
    K = dcfg.n_codebooks
    monkeypatch.setenv("PTTS_DAC_TC", "1")
    _, tc = m._encode(wav[:, 0], K, return_latents=True)
    monkeypatch.setenv("PTTS_DAC_TC", "0")
    _, gen = m._encode(wav[:, 0], K, return_latents=True)
    a, b = tc.float().cpu().numpy(), gen.float().cpu().numpy()
    assert rms(a) > 1e-2
    assert rms(a - b) < 0.05 * rms(a), (rms(a - b), rms(a))


def _generate_model():
    from parler_tts_b200 import ParlerTTSConfig, ParlerTTSForConditionalGeneration
    cfg, dcfg = tiny_cfg(), encode_cfg()
    assert (dcfg.n_codebooks, dcfg.codebook_size) == (cfg.num_codebooks, cfg.codebook_size)
    pc = ParlerTTSConfig(vocab_size=cfg.text_vocab_size, text_encoder={}, audio_encoder=product_codec_config(dcfg),
                         decoder=product_decoder_config(cfg))
    m = ParlerTTSForConditionalGeneration(pc, device=DEV, dtype=torch.bfloat16)
    m.load_state_dict(make_decoder_weights(cfg, seed=13, head_std=0.5), dac_state_dict=weights(dcfg))
    return cfg, m


@pytest.mark.gpu
@pytest.mark.parametrize("B,gen", [(3, dict(do_sample=False)), (3, dict(do_sample=True, top_k=8, seed=3)),
                                   (34, dict(do_sample=True, temperature=0.9, seed=11))])
def test_generate_from_input_values_equals_generate_from_its_codes(B, gen):
    from tests.helpers import synth_inputs
    cfg, model = _generate_model()
    enc, enc_mask, _, _ = synth_inputs(cfg, B, 6, 0, seed=B)
    g = torch.Generator().manual_seed(B)
    wav = (0.3 * torch.randn(B, 1, 3 * 512 + 100, generator=g)).to(DEV)
    kw = dict(encoder_outputs=(enc.to(DEV),), attention_mask=enc_mask.to(DEV), max_new_tokens=10, return_codes=True, **gen)
    a_audio, a = model.generate(input_values=wav, padding_mask=torch.ones_like(wav, dtype=torch.bool), **kw)
    codes = model.audio_encoder.encode(wav).audio_codes
    b_audio, b = model.generate(decoder_input_ids=codes, **kw)
    assert torch.equal(a.audio_codes, b.audio_codes)
    assert torch.equal(a_audio, b_audio) and a.audios_length == b.audios_length
    assert torch.equal(a.audio_codes[:, :, :codes.shape[-1]], codes[0])   # the continuation begins with the prompt's frames
