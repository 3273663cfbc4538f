"""Dump what the library's weight walks compute on seeded synthetic weights, so that two builds of the library (PTTS_LIB) can be
compared bit for bit: DAC decode (equal and ragged frame_lengths) and encode (codes and latents) on the wgmma, the generic bf16
(PTTS_DAC_TC=0) and the fp32 walks, for the 44.1 kHz codec and two small ones that reach the other walks; ptts_op_linear2 on
every matrix tensor id, LayerNorm on and off, path 0 and 1, bf16 and f32 (a refused combination records its error message);
and the prefill logits, one multi-kernel decode step's logits and teacher-forced scoring of two decoder shapes.
Usage: python tools/abi_bitwise.py dump OUT.npz
       python tools/abi_bitwise.py compare A.npz B.npz"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
DAC_PATHS = {"tc": ("bf16", "1"), "generic": ("bf16", "0"), "f32": ("f32", "1")}
# tensor id -> (K is ffn_dim, epilogue: 0 store, 1 act, 2 residual, 3 f32 logits)
MATRIX_IDS = {4: (0, 0), 5: (0, 0), 6: (0, 0), 7: (0, 2), 10: (0, 0), 11: (0, 0), 12: (0, 0), 13: (0, 2), 16: (0, 1), 17: (1, 2),
              20: (0, 3)}


def codecs():
    from oracle.config import dac_cfg, tiny_dac_cfg
    return {
        "44k": (dac_cfg(), 131, [131, 129, 16, 1, 0], 44100 + 123),
        # widths the wgmma kernel declines: the generic walks in bf16 as well
        "tiny": (tiny_dac_cfg(encoder_hidden_size=8), 40, [40, 17, 1, 0, 33], 3 * 512 + 100),
        # the wgmma decode walk with its generic output conv (1024 channels: past the one-thread-per-sample kernel)
        "wide": (tiny_dac_cfg(decoder_hidden_size=2048, upsampling_ratios=[4], encoder_hidden_size=64, downsampling_ratios=[4]),
                 40, [40, 17, 1, 0, 33], 1003),
    }


def dump_codecs(out):
    import torch
    from parler_tts_b200 import DACConfig, DACModel
    from oracle.weights import make_dac_weights
    from tests.dac_encode_oracle import make_dac_encoder_weights
    for name, (d, T, lengths, samples) in codecs().items():
        cfg = DACConfig(num_codebooks=d.n_codebooks, codebook_size=d.codebook_size, latent_dim=d.hidden_size, codebook_dim=d.codebook_dim,
                        decoder_dim=d.decoder_hidden_size, decoder_rates=tuple(d.upsampling_ratios),
                        encoder_dim=d.get("encoder_hidden_size", 64), encoder_rates=tuple(d.get("downsampling_ratios", [2, 4, 8, 8])))
        w = make_dac_weights(d, seed=3)
        w.update(make_dac_encoder_weights(d, seed=7))
        g = torch.Generator().manual_seed(9)
        codes = torch.randint(0, d.codebook_size, (1, len(lengths), d.n_codebooks, T), generator=g).to(DEV)
        wav = (0.3 * torch.randn(2, 1, samples, generator=g)).to(DEV)
        for path, (dt, tc) in DAC_PATHS.items():
            os.environ["PTTS_DAC_TC"] = tc
            m = DACModel(cfg, DEV, torch.bfloat16 if dt == "bf16" else torch.float32).load_state_dict(w)
            out[f"dac/{name}/{path}/decode"] = m.decode(codes).audio_values
            out[f"dac/{name}/{path}/decode_ragged"] = m.decode(codes, frame_lengths=lengths).audio_values
            c, lat = m._encode(wav[:, 0], d.n_codebooks, return_latents=True)
            out[f"dac/{name}/{path}/encode_codes"] = c
            out[f"dac/{name}/{path}/encode_latents"] = lat
    os.environ.pop("PTTS_DAC_TC", None)


def decoder_shapes():
    from oracle.config import decoder_cfg
    return {"mini": decoder_cfg(num_hidden_layers=2, max_position_embeddings=160),
            "gqa": decoder_cfg(hidden_size=256, num_attention_heads=4, num_key_value_heads=2, num_cross_attention_key_value_heads=1,
                               ffn_dim=1024, num_hidden_layers=2, max_position_embeddings=160, activation_function="silu")}


def dump_decoders(out):
    import torch
    from parler_tts_b200 import _lib
    from parler_tts_b200.modeling import DecoderEngine
    from oracle.weights import make_decoder_weights
    from tests.helpers import product_decoder_config, synth_inputs
    lib = _lib.lib()
    for name, cfg in decoder_shapes().items():
        w = make_decoder_weights(cfg, seed=5, head_std=0.2)
        g = torch.Generator().manual_seed(6)
        for k in w:   # LayerNorms far from the identity, so that a wrong gamma, beta or folded vector shows
            if "layer_norm" in k:
                w[k] = torch.exp(torch.randn(w[k].shape, generator=g)) if k.endswith(".weight") else torch.randn(w[k].shape, generator=g)
        H, F, V, K = cfg.hidden_size, cfg.ffn_dim, cfg.vocab_size, cfg.num_codebooks
        N = {4: (cfg.num_attention_heads + 2 * cfg.num_key_value_heads) * 64, 7: H, 10: H,
             11: 2 * cfg.num_cross_attention_key_value_heads * 64, 13: H, 16: F, 17: H, 20: K * V}
        N[5] = N[6] = N[4]
        N[12] = N[11]
        for dt in (torch.bfloat16, torch.float32):
            eng = DecoderEngine(product_decoder_config(cfg), DEV, dt).load_state_dict(w)
            tag = f"{name}/{'bf16' if dt == torch.bfloat16 else 'f32'}"
            for tid, (k_is_f, epi) in MATRIX_IDS.items():
                Kd = F if k_is_f else H
                for index in ((0, 1) if tid == 20 else (1,)):
                    for M in (33, 256):
                        x = torch.randn(M, Kd, generator=g).to(DEV, dt)
                        res = torch.randn(M, N[tid], generator=g).to(DEV, dt) if epi == 2 else None
                        for use_ln in (0, 1):
                            for path in (0, 1):
                                y = torch.full((M, N[tid]), float("nan"), device=DEV,
                                               dtype=torch.float32 if epi == 3 or dt == torch.float32 else torch.bfloat16)
                                stats = torch.empty(2 * M, dtype=torch.float32, device=DEV)
                                key = f"linear/{tag}/t{tid}/i{index}/M{M}/ln{use_ln}/p{path}"
                                e = lib.ptts_op_linear2(C.byref(eng.c), _lib.ptr(eng.blob), tid, index, _lib.ptr(x), M, use_ln, epi,
                                                        _lib.ptr(res), _lib.ptr(y), path, _lib.ptr(stats), _lib.stream_ptr())
                                out[key] = y if e == 0 else np.frombuffer(lib.ptts_last_error(), dtype=np.uint8)
            B, S, P, L, T = 32, 24, 16, 6, 5
            enc, em, pr, pm = synth_inputs(cfg, B, S, P, seed=4)
            os.environ["PTTS_FUSED"] = "0"   # the multi-kernel decode step: the decode GEMMs through run_forward
            sess = eng.session(B, P, S, P + L + 2, max_input_len=T)
            sess.begin(L, do_sample=False)
            sess.prefill(pr, pm, enc, em)
            out[f"prefill/{tag}/logits"] = sess.logits.clone()
            sess.sample()
            sess.decode_forward()
            out[f"decode/{tag}/logits"] = sess.logits.clone()
            os.environ.pop("PTTS_FUSED")
            ids = torch.randint(0, V, (B * K, T), generator=g)
            labels = torch.randint(0, V, (B, T, K), generator=g)
            nll = torch.empty(B, T, K, dtype=torch.float32, device=DEV)
            sess.score(pr, pm, enc, em, ids, labels, nll)
            out[f"score/{tag}/nll"] = nll
            logits = torch.empty(B * K, T, V, dtype=torch.float32, device=DEV)
            sess.score(pr, pm, enc, em, ids, None, None, logits=logits)
            out[f"score/{tag}/logits"] = logits
            del sess, eng
            torch.cuda.empty_cache()


def dump(path):
    import torch
    sys.path.insert(0, ROOT)
    out = {}
    dump_codecs(out)
    dump_decoders(out)
    torch.cuda.synchronize()
    arrays = {}
    for k, v in out.items():
        if isinstance(v, torch.Tensor):
            v = v.detach().cpu()
            v = v.view(torch.int16).numpy() if v.dtype == torch.bfloat16 else v.numpy()
        arrays[k] = v
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    np.savez(path, **arrays)
    refused = sum(1 for v in arrays.values() if v.dtype == np.uint8)
    print(f"{path}: {len(arrays)} arrays ({refused} refused linear calls), lib {os.environ.get('PTTS_LIB', '(product)')}")


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    ok = set(a.files) == set(b.files)
    if not ok:
        print("different keys:", sorted(set(a.files) ^ set(b.files))[:10])
    same = 0
    for k in sorted(set(a.files) & set(b.files)):
        if a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)):
            same += 1
        else:
            ok = False
            print(f"{k}: DIFFERENT (shapes {a[k].shape} / {b[k].shape})")
    print(f"{same} of {len(a.files)} arrays bitwise identical")
    print("BITWISE", "OK" if ok else "FAILED")
    return ok


if __name__ == "__main__":
    if sys.argv[1] == "dump":
        dump(sys.argv[2])
    else:
        sys.exit(0 if compare(sys.argv[2], sys.argv[3]) else 1)
