"""DAC encode timing (waveform -> codes) at the 44.1 kHz DAC shape: B = 32 prompts of 5 s, bf16, wgmma path.

After warm-up it reports
  * the whole DACModel.encode call (CUDA events, median of REPS calls): ms, x real time, achieved TFLOP/s;
  * the encoder convolutions and the quantizer separately: device time per call summed by kernel name from a torch.profiler
    run of its own (quantize_kernel vs every other kernel of the call), with TFLOP/s from each part's FLOP count;
  * the time generate(input_values=w) adds over generate(decoder_input_ids=codes) at the same shapes (Parler-TTS-Mini, bf16,
    the bench's prompt and description lengths, 32 new tokens; host clock around synchronised calls, median);
  * the card name and power limit, read in the same run.
FLOPs are counted from the config below (2 per multiply-add, the strided convs at their k = 2s size, not the 1.5x the
super-row rewrite executes).  Writes $PTTS_TOOLS_OUT/dac_encode_bench.json (default tools_out/) and prints it.
Usage: python tools/bench_dac_encode.py [B] [seconds]
"""
import json
import math
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from oracle.config import dac_cfg
from oracle.weights import make_dac_weights
from tests.dac_encode_oracle import make_dac_encoder_weights
from parler_tts_b200 import DACConfig, ParlerTTSConfig, ParlerTTSDecoderConfig, ParlerTTSForConditionalGeneration

REPS = 5


def encode_flops_per_frame(c: DACConfig) -> dict:
    """Multiply-adds x 2 per code frame (hop samples) of the encoder convs and of the residual quantizer."""
    hop = math.prod(c.encoder_rates)
    rows, C = hop, c.encoder_dim
    conv = 2 * 7 * C * rows                                      # input conv, 1 -> C
    for s in c.encoder_rates:
        conv += 3 * 2 * (7 * C * C + C * C) * rows                # residual units: k7 + k1
        conv += 2 * (2 * s * C) * (2 * C) * (rows // s)           # Conv1d(C -> 2C, k = 2s, stride s)
        rows //= s
        C *= 2
    conv += 2 * 3 * C * c.latent_dim * rows                      # final k3 conv
    K, D, Z, cs = c.num_codebooks, c.codebook_dim, c.latent_dim, c.codebook_size
    quant = K * 2 * (D * Z + cs * D + Z * D)                     # in_proj, cosine against every code, out_proj
    return {"encoder_convs": conv, "quantizer": quant}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    secs = float(sys.argv[2]) if len(sys.argv) > 2 else 5.0
    dev = torch.device("cuda", 0)
    os.environ["PTTS_DAC_TC"] = "1"
    cfg = ParlerTTSConfig(vocab_size=32128, text_encoder={}, audio_encoder=DACConfig(), decoder=ParlerTTSDecoderConfig(**bench.MINI))
    model = ParlerTTSForConditionalGeneration(cfg, device=dev, dtype=torch.bfloat16)
    model.load_state_dict(bench.synthetic_state_dict(bench.MINI, dev))
    dw = make_dac_weights(dac_cfg(), seed=3)
    dw.update(make_dac_encoder_weights(dac_cfg(), seed=7))
    model.audio_encoder.load_state_dict(dw)
    codec = model.audio_encoder
    n = int(secs * cfg.audio_encoder.sampling_rate)
    g = torch.Generator().manual_seed(0)
    t = torch.arange(n) / cfg.audio_encoder.sampling_rate
    wav = (0.3 * torch.sin(2 * math.pi * 200.0 * t) + 0.1 * torch.randn(B, n, generator=g))[:, None, :].to(dev)
    frames = math.ceil(n / codec.hop_length)
    fl = encode_flops_per_frame(cfg.audio_encoder)

    for _ in range(3):
        codec.encode(wav)
    torch.cuda.synchronize()
    ms = []
    for _ in range(REPS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        codes = codec.encode(wav).audio_codes
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    call_ms = statistics.median(ms)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(REPS):
            codec.encode(wav)
        torch.cuda.synchronize()
    part_us = {"encoder_convs": 0.0, "quantizer": 0.0}
    for ev in prof.key_averages():
        dt = getattr(ev, "device_time_total", None)
        if dt is None:
            dt = ev.cuda_time_total
        if dt <= 0 or "memcpy" in ev.key.lower() or "memset" in ev.key.lower():
            continue
        part_us["quantizer" if "quantize_kernel" in ev.key else "encoder_convs"] += dt / REPS

    total_flop = (fl["encoder_convs"] + fl["quantizer"]) * B * frames
    audio_s = B * n / cfg.audio_encoder.sampling_rate
    out = {"card": card(), "B": B, "seconds": secs, "frames": frames,
           "gflop_per_frame": {k: v / 1e9 for k, v in fl.items()},
           "encode_call": {"ms": call_ms, "x_real_time": audio_s / (call_ms / 1e3), "tflops": total_flop / (call_ms / 1e3) / 1e12},
           "parts": {k: {"ms": us / 1e3, "tflops": fl[k] * B * frames / (us / 1e6) / 1e12 if us > 0 else None} for k, us in part_us.items()}}

    # generate(input_values=w) vs generate(decoder_input_ids=codes), same shapes and seed
    enc, em, pr, pm = bench.synthetic_inputs(B, 1024, 1, device=dev)
    kw = dict(encoder_outputs=(enc,), attention_mask=em, prompt_hidden_states=pr, prompt_attention_mask=pm, max_new_tokens=32,
              do_sample=True, top_k=50, seed=1)

    def timed(**extra):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.generate(**kw, **extra)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    timed(input_values=wav), timed(decoder_input_ids=codes)
    a, b = [], []
    for _ in range(REPS):   # alternate the two, so drift hits both alike
        a.append(timed(input_values=wav))
        b.append(timed(decoder_input_ids=codes))
    out["generate"] = {"input_values_ms": statistics.median(a), "decoder_input_ids_ms": statistics.median(b),
                       "added_ms": statistics.median(a) - statistics.median(b), "max_new_tokens": 32}
    out["card_after"] = card()
    print(json.dumps(out))
    out_dir = os.environ.get("PTTS_TOOLS_OUT", os.path.join(ROOT, "tools_out"))
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "dac_encode_bench.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
