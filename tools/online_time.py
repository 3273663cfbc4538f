"""Online continuous batching under Poisson arrivals: Parler-TTS-Mini, bf16, the workload of tools/continuous_time.py (the bench's
synthetic weights, prompt and description lengths, top-k 50, max_new_tokens 1720, EOS bias +1.5, the value that tool's calibration
found) through a ContinuousEngine (batch_size 32, refill_every 16, stream=True).
First, generate_continuous(stream=True) over the whole list (all N requests known up front) gives the offline audio per wall second
and request rate R0.  Then, for each arrival rate in RATES x R0, seeded Poisson arrivals: the loop submits the requests due before
each step() (and sleeps while the engine is idle and the next one is not due yet), until every request has ended.  Per request:
  admission delay -- from its submit() to the return of the step() that admitted it into a slot;
  first audio     -- from its submit() to the return of the step() that yielded its first event (the chunk's codec call is
                     enqueued by then; it completes one codec call later);
  completion      -- from its submit() to the return of the step() that yielded its final event.
Reported as p50 / p90 / p99 in ms, with decoded audio per wall second (the whole run, first submit to a device synchronise after the
last step).  Host clock (time.perf_counter).
Usage: python tools/online_time.py [N]
Writes tools_out/online_time.json (or $PTTS_TOOLS_OUT/...) with the card's name, power limit and max SM clock.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from parler_tts_b200 import DACConfig, ParlerTTSConfig, ParlerTTSDecoderConfig, ParlerTTSForConditionalGeneration

N = int(sys.argv[1]) if len(sys.argv) > 1 else 256
RATES, BATCH, REFILL, MAX_NEW, BIAS = (0.5, 0.8, 1.0, 1.2), 32, 16, 1720, 1.5
if not torch.cuda.is_available():
    sys.exit("online_time.py measures on the GPU; none is available")
dev = torch.device("cuda", 0)
cfg = ParlerTTSConfig(vocab_size=32128, text_encoder={}, audio_encoder=DACConfig(), decoder=ParlerTTSDecoderConfig(**bench.MINI))
model = ParlerTTSForConditionalGeneration(cfg, device=dev, dtype=torch.bfloat16)
model.load_state_dict(bench.synthetic_state_dict(bench.MINI, dev))
model.audio_encoder.load_state_dict(bench.synth_dac_weights(cfg.audio_encoder, dev))
d = cfg.decoder
P, S, eos, sr = bench.P_LEN, bench.S_LEN, d.eos_token_id, cfg.audio_encoder.sampling_rate
enc, em, pr, pm = (t.to(dev) for t in bench.synthetic_inputs(N, 1024, 1))
kw = dict(do_sample=True, top_k=50, seed=3, max_new_tokens=MAX_NEW, sequence_bias={(eos,): BIAS})


def offline():
    """generate_continuous over the whole list: (wall s, decoded samples)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run = model.generate_continuous(encoder_outputs=(enc,), attention_mask=em, prompt_hidden_states=pr, prompt_attention_mask=pm,
                                    batch_size=BATCH, refill_every=REFILL, stream=True, **kw)
    samples = sum(chunk.shape[0] for _, chunk, final in run if chunk.numel() > 1 or not final)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, samples


def online(rate, seed):
    """One Poisson-arrival run at `rate` requests per second: per-request latencies (s) and (wall s, decoded samples)."""
    arrive = np.cumsum(np.random.default_rng(seed).exponential(1.0 / rate, N))
    engine = model.continuous_engine(batch_size=BATCH, refill_every=REFILL, max_description_length=S, max_prompt_length=P,
                                     stream=True, **kw)
    sub, adm, first, done = {}, {}, {}, {}
    samples, nxt, queued = 0, 0, set()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    while nxt < N or not engine.idle:
        now = time.perf_counter() - t0
        if engine.idle and nxt < N and arrive[nxt] > now:
            time.sleep(arrive[nxt] - now)
            now = time.perf_counter() - t0
        while nxt < N and arrive[nxt] <= now:
            i = nxt
            assert engine.submit(encoder_outputs=(enc[i:i + 1],), attention_mask=em[i:i + 1], prompt_hidden_states=pr[i:i + 1],
                                 prompt_attention_mask=pm[i:i + 1]) == i
            sub[i] = time.perf_counter() - t0
            queued.add(i)
            nxt += 1
        events = engine.step()
        t = time.perf_counter() - t0
        for i in [i for i in queued if engine._status[i] != engine.QUEUED]:
            adm[i] = t
            queued.discard(i)
        for r, chunk, final in events:
            first.setdefault(r, t)
            if final:
                done[r] = t
            if chunk.numel() > 1 or not final:
                samples += chunk.shape[0]
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    lat = lambda m: [m[i] - sub[i] for i in range(N)]
    return dict(admission=lat(adm), first_audio=lat(first), completion=lat(done)), (wall, samples)


pct = lambda v: {f"p{q}": round(float(np.percentile(np.asarray(v) * 1e3, q)), 1) for q in (50, 90, 99)}
offline()                                                    # warm-up: every shape the runs take
wall0, samples0 = offline()
r0 = N / wall0
online(r0, 0)                                                # warm-up of the engine's loop
res = dict(offline=dict(wall_s=round(wall0, 3), requests_per_s=round(r0, 2), audio_s_per_wall_s=round(samples0 / sr / wall0, 3)))
for x in RATES:
    lats, (wall, samples) = online(x * r0, 1)
    res[f"{x}x"] = dict(rate_per_s=round(x * r0, 2), wall_s=round(wall, 3), audio_s_per_wall_s=round(samples / sr / wall, 3),
                        **{k: pct(v) for k, v in lats.items()})
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
r = dict(card=smi, N=N, P=P, S=S, batch_size=BATCH, refill_every=REFILL, eos_bias=BIAS, audio_s_total=samples0 / sr, runs=res)
print(json.dumps(r), flush=True)
out_dir = os.environ.get("PTTS_TOOLS_OUT", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools_out"))
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "online_time.json"), "w") as f:
    json.dump(r, f, indent=1)
