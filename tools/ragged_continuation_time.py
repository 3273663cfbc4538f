"""Cost of a ragged continuation (generate(decoder_input_ids, decoder_attention_mask)) on the bench workload: Parler-TTS-Mini,
bf16, B = 32, the bench's prompt and description lengths, code prefixes spread from 0.5 s to 5 s (43 .. 430 frames at 86 Hz).
Times, on a host clock around calls that end in a device synchronise (median of REPS after one warm-up call):
  * ragged   -- one generate() call over the 32 prefixes of different lengths;
  * singles  -- the 32 generate() calls of one utterance each that it replaces;
  * uniform  -- one generate() call with every row at the longest prefix;
and, with CUDA events, the mean decode step (32 steps after the first column) of the ragged session against a uniform session of
the same n0.  Every call generates NEW columns (min_new_tokens = max_new_tokens, special ids suppressed).
Usage: python tools/ragged_continuation_time.py [new_tokens]   (default 64)
Writes tools_out/ragged_continuation_time.json (or $PTTS_TOOLS_OUT/...) with the card's name, power limit and max SM clock.
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
from parler_tts_b200.modeling import prepare_ragged_decoder_input_ids

NEW = int(sys.argv[1]) if len(sys.argv) > 1 else 64
REPS, STEPS = 3, 32
dev = torch.device("cuda", 0)
cfg = ParlerTTSConfig(vocab_size=32128, text_encoder={}, audio_encoder=DACConfig(), decoder=ParlerTTSDecoderConfig(**bench.MINI))
model = ParlerTTSForConditionalGeneration(cfg, device=dev, dtype=torch.bfloat16)
model.load_state_dict(bench.synthetic_state_dict(bench.MINI, dev))
model.audio_encoder.load_state_dict(bench.synth_dac_weights(cfg.audio_encoder, dev))
d = cfg.decoder
B, K, P, S = 32, d.num_codebooks, bench.P_LEN, bench.S_LEN
enc, em, pr, pm = bench.synthetic_inputs(B, 1024, 1, device=dev)
lens = [43 + (430 - 43) * b // (B - 1) for b in range(B)]
N = max(lens)
codes = torch.randint(0, 1024, (B, K, N), generator=torch.Generator().manual_seed(1)).to(dev)
mask = (torch.arange(N)[None, :] < torch.tensor(lens)[:, None]).long().to(dev)
kw = dict(do_sample=True, top_k=50, max_new_tokens=NEW, min_new_tokens=NEW, _suppress_special=True, return_codes=True)


def call(lo, hi, **extra):
    return model.generate(encoder_outputs=(enc[lo:hi],), attention_mask=em[lo:hi], prompt_hidden_states=pr[lo:hi],
                          prompt_attention_mask=pm[lo:hi], **kw, **extra)


def timed(fn):
    ts = []
    for rep in range(REPS + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        if rep > 0:
            ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


ragged_ms = timed(lambda: call(0, B, decoder_input_ids=codes, decoder_attention_mask=mask))
singles_ms = timed(lambda: [call(b, b + 1, decoder_input_ids=codes[b:b + 1, :, :lens[b]], row_base=b * K) for b in range(B)])
uniform_ms = timed(lambda: call(0, B, decoder_input_ids=codes))


def step_ms(input_lens):
    """Mean decode step of a session that continues from the [B * K, n0] input (with input_lens: ragged), CUDA events."""
    ids, il = prepare_ragged_decoder_input_ids(codes, mask if input_lens else torch.ones_like(mask), B, K, d.vocab_size,
                                               d.bos_token_id, dev)
    n0 = ids.shape[1]
    L = n0 + STEPS + 1
    sess = model.decoder.engine.session(B, P, S, P + L, max_input_len=n0)
    ts = []
    for rep in range(REPS + 1):
        sess.begin(L, do_sample=True, top_k=50, seed=rep, min_new_tokens=L, suppress_special=True, codebook_size=1024, input_ids=ids,
                   input_lens=il if input_lens else None)
        sess.prefill(pr, pm, enc, em)
        sess.sample()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        sess.decode_steps(STEPS)
        ev[1].record()
        torch.cuda.synchronize()
        if rep > 0:
            ts.append(ev[0].elapsed_time(ev[1]) / STEPS)
    return statistics.median(ts), n0, sess.fused


rag_step, n0, kind_r = step_ms(True)
uni_step, _, kind_u = step_ms(False)
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
r = dict(card=smi, B=B, P=P, S=S, new_tokens=NEW, prefix_frames=lens, ragged_call_ms=ragged_ms, single_calls_ms=singles_ms,
         uniform_call_at_longest_ms=uniform_ms, n0=n0, ragged_decode_step_ms=rag_step, uniform_decode_step_ms=uni_step,
         step_kernel_kind=(kind_r, kind_u))
print(json.dumps(r), flush=True)
out_dir = os.environ.get("PTTS_TOOLS_OUT", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools_out"))
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "ragged_continuation_time.json"), "w") as f:
    json.dump(r, f, indent=1)
