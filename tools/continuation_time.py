"""Cost of continuing from audio codes (generate(decoder_input_ids=...)) on the bench workload: Parler-TTS-Mini, bf16, B = 32, the
bench's prompt and description lengths.  For each prefix of n frames (n0 = n + 1 input columns, n = 0 is a plain generate()) it
times, with CUDA events over several repetitions (median):
  * prefill        -- ptts_prefill: prompt prefix + n0 columns through the decoder in one pass, cross K/V projected once;
  * first column   -- begin + prefill + the first sample: time to the first new token column;
  * decode step    -- the mean of 32 decode steps after it (the cached length grows with n).
Usage: python tools/continuation_time.py [frames ...]   (default 0 86 430 1720; 86 frames are 1 s at 86 Hz)
Writes tools_out/continuation_time.json (or $PTTS_TOOLS_OUT/continuation_time.json) and prints one line per prefix.
"""
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from parler_tts_b200 import DACConfig, ParlerTTSConfig, ParlerTTSDecoderConfig, ParlerTTSForConditionalGeneration
from parler_tts_b200.modeling import prepare_decoder_input_ids

frames = [int(a) for a in sys.argv[1:]] or [0, 86, 430, 1720]
dev = torch.device("cuda", 0)
cfg = ParlerTTSConfig(vocab_size=32128, text_encoder={}, audio_encoder=DACConfig(), decoder=ParlerTTSDecoderConfig(**bench.MINI))
model = ParlerTTSForConditionalGeneration(cfg, device=dev, dtype=torch.bfloat16)
model.load_state_dict(bench.synthetic_state_dict(bench.MINI, dev))
d = cfg.decoder
B, K, P, S, STEPS, REPS = 32, d.num_codebooks, bench.P_LEN, bench.S_LEN, 32, 5
enc, em, pr, pm = bench.synthetic_inputs(B, 1024, 1, device=dev)
gen = dict(do_sample=True, top_k=50, suppress_special=True, codebook_size=1024)
rows = []
for n in frames:
    if P + n + 1 + STEPS + 1 > d.max_position_embeddings:
        print(f"skip {n} frames: {P} + {n + 1} + {STEPS + 1} positions exceed {d.max_position_embeddings}", flush=True)
        continue
    ids = None
    if n > 0:
        codes = torch.randint(0, 1024, (B * K, n), generator=torch.Generator().manual_seed(n))
        ids = prepare_decoder_input_ids(codes, B, K, d.vocab_size, d.bos_token_id, dev)
    n0 = 1 if ids is None else ids.shape[1]
    L = n0 + STEPS + 1
    sess = model.decoder.engine.session(B, P, S, P + L, max_input_len=n0)
    t_pre, t_first, t_step = [], [], []
    for rep in range(REPS + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        torch.cuda.synchronize()
        ev[0].record()
        sess.begin(L, seed=1 + rep, min_new_tokens=L, input_ids=ids, **gen)
        ev[1].record()
        sess.prefill(pr, pm, enc, em)
        ev[2].record()
        sess.sample()
        ev[3].record()
        sess.decode_steps(STEPS)
        ev[4].record()
        torch.cuda.synchronize()
        if rep == 0:
            continue   # first call: session set-up, lazy module loads
        t_pre.append(ev[1].elapsed_time(ev[2]))
        t_first.append(ev[0].elapsed_time(ev[3]))
        t_step.append(ev[3].elapsed_time(ev[4]) / STEPS)
    r = dict(frames=n, n0=n0, prefill_rows=B * (P + n0), prefill_ms=statistics.median(t_pre), first_column_ms=statistics.median(t_first),
             decode_step_ms=statistics.median(t_step), fused=sess.fused)
    rows.append(r)
    print(f"frames {n:5d} (n0 {n0:5d}, {r['prefill_rows']:6d} prefill rows): prefill {r['prefill_ms']:8.2f} ms, first column "
          f"{r['first_column_ms']:8.2f} ms, decode step {r['decode_step_ms'] * 1e3:7.0f} us (step kernel kind {r['fused']})", flush=True)
out_dir = os.environ.get("PTTS_TOOLS_OUT", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools_out"))
os.makedirs(out_dir, exist_ok=True)
props = torch.cuda.get_device_properties(dev)
with open(os.path.join(out_dir, "continuation_time.json"), "w") as f:
    json.dump(dict(device=props.name, B=B, P=P, S=S, rows=rows), f, indent=1)
