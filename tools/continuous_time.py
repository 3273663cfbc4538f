"""What continuous batching gives back on a mixed-length workload: Parler-TTS-Mini, bf16, N requests (default 256) with the bench's
prompt and description lengths, whose lengths spread over about 1 .. 20 s (max_new_tokens 1720 frames at 86 Hz) through a single-id
sequence_bias on EOS.  The bias is calibrated first on 32 requests: bracketed, then bisected until the median request ends between
5 and 15 s.  The tool stops with an error when no bias does that, or when the run's requests do not spread (the longest under 4x
the shortest): a workload without the mix says nothing about the feature.
Alternating runs, REPS of each after one warm-up of each:
  * static     -- generate() over all N requests (shards of 32, each running to its longest request);
  * continuous -- generate_continuous(batch_size=32, refill_every=R) for R in {8, 16, 32}, the run consumed to the end;
each timed on a host clock around the whole call ending in a device synchronise.  Reported: audio seconds per wall second, and the
refill cost per boundary = (continuous wall time - its decode steps x the slot-mode decode step) / its boundaries, with the step
timed by CUDA events over 64 steps of a 32-slot session in slot mode.
Usage: python tools/continuous_time.py [N]
Writes tools_out/continuous_time.json (or $PTTS_TOOLS_OUT/...) with the card's name, power limit and max SM clock.
"""
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from parler_tts_b200 import DACConfig, ParlerTTSConfig, ParlerTTSDecoderConfig, ParlerTTSForConditionalGeneration
from parler_tts_b200.modeling import GenSession

N = int(sys.argv[1]) if len(sys.argv) > 1 else 256
REPS, REFILLS, MAX_NEW = 2, (8, 16, 32), 1720
dev = torch.device("cuda", 0)
cfg = ParlerTTSConfig(vocab_size=32128, text_encoder={}, audio_encoder=DACConfig(), decoder=ParlerTTSDecoderConfig(**bench.MINI))
model = ParlerTTSForConditionalGeneration(cfg, device=dev, dtype=torch.bfloat16)
model.load_state_dict(bench.synthetic_state_dict(bench.MINI, dev))
model.audio_encoder.load_state_dict(bench.synth_dac_weights(cfg.audio_encoder, dev))
d = cfg.decoder
K, P, S, eos = d.num_codebooks, bench.P_LEN, bench.S_LEN, d.eos_token_id
enc, em, pr, pm = (t.to(dev) for t in bench.synthetic_inputs(N, 1024, 1))
inputs = dict(encoder_outputs=(enc,), attention_mask=em, prompt_hidden_states=pr, prompt_attention_mask=pm)
base = dict(do_sample=True, top_k=50, seed=3, max_new_tokens=MAX_NEW)


def ends(raw):
    """Columns of each request's EOS in its last codebook (MAX_NEW + 1 where it ran to the limit)."""
    last = raw.view(-1, K, raw.shape[1])[:, -1] == eos
    return torch.where(last.any(-1), last.int().argmax(-1) + 1, torch.full_like(last[:, 0], MAX_NEW + 1, dtype=torch.long)).tolist()


def median_end(bias):
    probe = model.generate(encoder_outputs=(enc[:32],), attention_mask=em[:32], prompt_hidden_states=pr[:32], prompt_attention_mask=pm[:32],
                           return_dict_in_generate=True, sequence_bias={(eos,): float(bias)}, **base)
    return statistics.median(ends(probe.raw_ids))


LO, HI = 430, 1290          # 5 .. 15 s of frames: where the calibration wants the median request to end
tried = {}                  # bias -> median end column; the end falls as the bias grows


def probe(b):
    m = tried[b] = median_end(b)
    return m


bias, b = None, 0.0
m = probe(b)
lo, hi = (b, None) if m > HI else (None, b)     # lo: ends too late, hi: too early
if LO <= m <= HI:
    bias = b
step = 2.0
while bias is None and (lo is None or hi is None) and len(tried) < 10:   # bracket: steps that double
    b = lo + step if hi is None else hi - step
    m = probe(b)
    if LO <= m <= HI:
        bias = b
    elif m > HI:
        lo = b
    else:
        hi = b
    step *= 2
for _ in range(12):                                                          # then bisect the bracket
    if bias is not None or lo is None or hi is None:
        break
    b = (lo + hi) / 2
    m = probe(b)
    if LO <= m <= HI:
        bias = b
    elif m > HI:
        lo = b
    else:
        hi = b
if bias is None:
    sys.exit(f"no EOS bias gives a median request of 5 .. 15 s (median end column per bias tried: {tried})")
kw = dict(base, sequence_bias={(eos,): bias})


lengths_s = None


def static():
    global lengths_s
    out = model.generate(**inputs, return_dict_in_generate=True, **kw)
    lengths_s = sorted(round(e / 86.13, 2) for e in ends(out.raw_ids))
    return sum(out.audios_length)


def continuous(refill):
    run = model.generate_continuous(**inputs, batch_size=32, refill_every=refill, **kw)
    total = sum(w.shape[0] for _, w in run)
    return total, run


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


# the slot-mode decode step: 64 steps of a 32-slot session after set_slots, CUDA events
sess = GenSession(model.decoder.engine, 32, P, S, P + 80, max_input_len=2)
steps_ms = []
for rep in range(REPS + 1):
    sess.begin(70, do_sample=True, top_k=50, seed=rep, min_new_tokens=70, suppress_special=True, codebook_size=1024)
    sess.prefill(pr[:32], pm[:32], enc[:32], em[:32])
    sess.sample()
    sess.set_slots(2, [0] * 32, list(range(32)))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    sess.decode_steps(64)
    ev[1].record()
    torch.cuda.synchronize()
    if rep > 0:
        steps_ms.append(ev[0].elapsed_time(ev[1]) / 64)
step_ms = statistics.median(steps_ms)
sess.close()

sr = cfg.audio_encoder.sampling_rate
res = {"static": []} | {f"continuous_{r}": [] for r in REFILLS}
boundary = {r: [] for r in REFILLS}
samples = None
for rep in range(REPS + 1):   # alternating; rep 0 warms every shape up
    ms, n = timed(static)
    samples = n
    if rep > 0:
        res["static"].append(n / sr / (ms / 1e3))
    for r in REFILLS:
        ms, (n, run) = timed(lambda: continuous(r))
        if rep > 0:
            res[f"continuous_{r}"].append(n / sr / (ms / 1e3))
            boundary[r].append((ms - run.steps * step_ms) / max(run.boundaries, 1))
if lengths_s[-1] < 4 * lengths_s[0]:
    sys.exit(f"the requests do not spread: {lengths_s[0]} .. {lengths_s[-1]} s at EOS bias {bias}")
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
r = dict(card=smi, N=N, P=P, S=S, eos_bias=bias, calibration=tried, audio_seconds_total=samples / sr, request_seconds=lengths_s,
         audio_s_per_wall_s={k: statistics.median(v) for k, v in res.items()}, runs=res, slot_step_ms=step_ms,
         refill_cost_ms_per_boundary={r: statistics.median(v) for r, v in boundary.items()})
print(json.dumps(r), flush=True)
out_dir = os.environ.get("PTTS_TOOLS_OUT", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools_out"))
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "continuous_time.json"), "w") as f:
    json.dump(r, f, indent=1)
