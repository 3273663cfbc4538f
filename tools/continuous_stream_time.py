"""What streaming costs and gives in continuous batching: generate_continuous(stream=True) against stream=False on the workload of
tools/continuous_time.py (Parler-TTS-Mini bf16, synthetic weights, N requests (default 256) with the bench's prompt and description
lengths, top-k 50, the EOS bias calibrated so the median request ends between 5 and 15 s), batch_size 32, refill_every 8 and 16.
Arms, alternated, REPS of each after one warm-up of each:
  * plain      -- stream=False;
  * stream     -- stream=True (ptts_dac_decode3: each layer computes only the rows the emitted samples need);
  * overlap    -- stream=True with DACModel._decode_windows replaced, here only, by a gather of each window to frame 0 and one
                  ragged ptts_dac_decode2 over them: the overlap-save decode that recomputes every layer over the whole window.
Reported:
  * decoded audio seconds per wall second (host clock around the whole run, ending in a device synchronise);
  * per-request time to first audio: a CUDA event recorded at each event the run yields (no sync in the consumer) against a start
    event recorded at the call, and against the request's admission (an event recorded when its slot import is enqueued; the first
    batch_size requests are admitted at the call).  For stream=False the request's only event is its first.  Median, p90, max;
  * the codec's device time for both window decodes on the windows of one captured boundary (the one with the most emitted
    frames), CUDA events over 20 calls;
  * the GFLOP those windows need, by arithmetic over the decoder's layers (not measured): every row of every window (overlap), the
    rows each layer needs (dac.cu window_margins), and those rounded out to 128-row tiles.
Usage: python tools/continuous_stream_time.py [N]
Writes tools_out/continuous_stream_time.json (or $PTTS_TOOLS_OUT/...) with the card's name, power limit and max SM clock.
"""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from parler_tts_b200 import DACConfig, DACModel, _lib, ParlerTTSConfig, ParlerTTSDecoderConfig, ParlerTTSForConditionalGeneration
from parler_tts_b200.modeling import GenSession

N = int(sys.argv[1]) if len(sys.argv) > 1 else 256
REPS, REFILLS, MAX_NEW, ARMS = 2, (8, 16), 1720, ("plain", "stream", "overlap")
dev = torch.device("cuda", 0)
cfg = ParlerTTSConfig(vocab_size=32128, text_encoder={}, audio_encoder=DACConfig(), decoder=ParlerTTSDecoderConfig(**bench.MINI))
model = ParlerTTSForConditionalGeneration(cfg, device=dev, dtype=torch.bfloat16)
model.load_state_dict(bench.synthetic_state_dict(bench.MINI, dev))
model.audio_encoder.load_state_dict(bench.synth_dac_weights(cfg.audio_encoder, dev))
dac = model.audio_encoder
K, eos, hop, sr = cfg.decoder.num_codebooks, cfg.decoder.eos_token_id, dac.hop_length, cfg.audio_encoder.sampling_rate
enc, em, pr, pm = (t.to(dev) for t in bench.synthetic_inputs(N, 1024, 1))
inputs = dict(encoder_outputs=(enc,), attention_mask=em, prompt_hidden_states=pr, prompt_attention_mask=pm)
base = dict(do_sample=True, top_k=50, seed=3, max_new_tokens=MAX_NEW)


# ---- the EOS bias: tools/continuous_time.py's calibration (bracket, then bisect, until the median request ends in 5 .. 15 s)
def median_end(bias):
    out = model.generate(encoder_outputs=(enc[:32],), attention_mask=em[:32], prompt_hidden_states=pr[:32], prompt_attention_mask=pm[:32],
                         return_dict_in_generate=True, sequence_bias={(eos,): float(bias)}, **base)
    last = out.raw_ids.view(-1, K, out.raw_ids.shape[1])[:, -1] == eos
    ends = torch.where(last.any(-1), last.int().argmax(-1) + 1, torch.full_like(last[:, 0], MAX_NEW + 1, dtype=torch.long))
    return statistics.median(ends.tolist())


LO, HI = 430, 1290
tried, bias, lo, hi, step = {}, None, None, None, 2.0
b = 0.0
while bias is None and len(tried) < 22:
    m = tried[b] = median_end(b)
    if LO <= m <= HI:
        bias = b
    elif m > HI:
        lo = b
    else:
        hi = b
    if bias is None:
        if lo is None or hi is None:
            b = lo + step if hi is None else hi - step
            step *= 2
        else:
            b = (lo + hi) / 2
if bias is None:
    sys.exit(f"no EOS bias gives a median request of 5 .. 15 s (median end column per bias tried: {tried})")
kw = dict(base, sequence_bias={(eos,): bias})


# ---- the overlap-save arm and the boundary capture -----------------------------------------------------------------------------
def overlap_windows(self, codes, windows):
    """Each window gathered to frame 0 and decoded whole by one ragged decode2 call; the caller keeps [lo, hi) of each row."""
    B, Kc, _ = codes.shape
    T = max(w[1] for w in windows)
    idx = torch.tensor([[min(s + f, codes.shape[2] - 1) for f in range(T)] for s, _, _, _ in windows], device=codes.device)
    gathered = torch.gather(codes, 2, idx[:, None, :].expand(B, Kc, T)).contiguous()
    lengths = torch.tensor([w[1] for w in windows], dtype=torch.int32).pin_memory().to(codes.device, non_blocking=True)
    need = C.c_int64()
    _lib.check(_lib.lib().ptts_dac_workspace_bytes(C.byref(self._c), B, T, C.byref(need)))
    if self._ws is None or self._ws.numel() < need.value:
        self._ws = torch.empty(need.value, dtype=torch.uint8, device=codes.device)
    audio = torch.empty(B, T * self.hop_length, dtype=self.dtype, device=codes.device)
    # ptts_dac_decode2 straight, as _decode_windows calls decode3: DACModel.decode's id range check would wait for the device
    _lib.check(_lib.lib().ptts_dac_decode2(C.byref(self._c), _lib.ptr(self.blob), _lib.ptr(self._ws), self._ws.numel(), _lib.ptr(gathered),
                                           B, T, _lib.ptr(lengths), _lib.ptr(audio), _lib.stream_ptr()))
    return audio


windowed = DACModel._decode_windows
captured = {}


def capturing(self, codes, windows):
    emit = sum(w[3] - w[2] for w in windows)
    if emit > captured.get("emit", -1):
        captured.update(emit=emit, codes=codes.clone(), windows=list(windows))
    return windowed(self, codes, windows)


admitted = []   # (event, rows) per slot import, in order
plain_import = GenSession.import_rows


def recording_import(self, src, src_rows, dst_rows):
    r = plain_import(self, src, src_rows, dst_rows)
    ev = torch.cuda.Event(enable_timing=True)
    ev.record()
    admitted.append((ev, len(dst_rows)))
    return r


GenSession.import_rows = recording_import


def run_arm(arm, refill, capture=False):
    DACModel._decode_windows = overlap_windows if arm == "overlap" else capturing if capture else windowed
    admitted.clear()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    start = torch.cuda.Event(enable_timing=True)
    start.record()
    run = model.generate_continuous(**inputs, batch_size=32, refill_every=refill, stream=arm != "plain", **kw)
    first, samples = {}, 0
    for ev in run:
        i, chunk = ev[0], ev[1]
        samples += chunk.shape[0]
        if i not in first:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            first[i] = e
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    DACModel._decode_windows = windowed
    adm = {}
    it = iter(admitted)
    ev, left = None, 0
    for _, req, _ in run.refills:
        while left == 0:
            ev, left = next(it)
        adm[req] = ev
        left -= 1
    from_call = [start.elapsed_time(first[i]) for i in range(N)]
    from_adm = [(adm[i].elapsed_time(first[i]) if i in adm else start.elapsed_time(first[i])) for i in range(N)]
    return samples / sr / wall, from_call, from_adm


def stats(v):
    v = sorted(v)
    return dict(median=statistics.median(v), p90=v[min(len(v) - 1, int(0.9 * len(v)))], max=v[-1])


res = {(a, r): [] for a in ARMS for r in REFILLS}
ttfa = {}
for rep in range(REPS + 1):   # alternated; rep 0 warms every shape up
    for r in REFILLS:
        for a in ARMS:
            rate, fc, fa = run_arm(a, r, capture=(rep == 1 and r == 16 and a == "stream"))
            if rep > 0:
                res[a, r].append(rate)
                ttfa.setdefault((a, r), (fc, fa))


# ---- codec time and arithmetic on the captured boundary ------------------------------------------------------------------------
def codec_ms(fn):
    for _ in range(3):
        fn(dac, captured["codes"], captured["windows"])
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(20):
        fn(dac, captured["codes"], captured["windows"])
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / 20


def layers(c):
    """(FLOP per output row, output rows per frame, taps reach (lo, hi) on the input, kind) for conv 1 .. output conv."""
    C, L = c.decoder_dim, [(2 * c.latent_dim * c.decoder_dim * 7, 1, "same", 3)]
    up = 1
    for i, s in enumerate(c.decoder_rates):
        cin, cout = C >> i, C >> (i + 1)
        up *= s
        L.append((2 * cin * cout * 2, up, "up", s))
        for d in (1, 3, 9):
            L += [(2 * cout * cout * 7, up, "same", 3 * d), (2 * cout * cout, up, "same", 0)]
    L.append((2 * (C >> len(c.decoder_rates)) * 7, up, "same", 3))
    return L


def margins(L):
    """dac.cu window_margins: each conv's output margins, walked back from the output conv."""
    out, lo, hi = [], 0, 0
    for flop, up, kind, r in reversed(L):
        out.append((lo, hi))
        if kind == "same":
            lo, hi = lo + r, hi + r
        else:
            s, pad = r, (r + 1) // 2
            lo, hi = 1 - ((pad - lo) // s), (hi - 1 + pad) // s + 1
    return out[::-1]


def gflop(windows, mode):
    L = layers(cfg.audio_encoder)
    M = margins(L)
    tot = 0
    for (flop, up, _, _), (mlo, mhi) in zip(L, M):
        for _, n, lo, hi in windows:
            if mode == "overlap":
                rows = n * up
            elif hi <= lo:
                rows = 0
            else:
                a, b = max(0, lo * up - mlo), min(n * up, hi * up + mhi)
                if mode == "tiles":
                    a, b = a // 128 * 128, min(n * up, -(-b // 128) * 128)
                rows = max(0, b - a)
            tot += rows * flop
    return tot / 1e9


codec = dict(windowed_ms=codec_ms(windowed), overlap_ms=codec_ms(overlap_windows),
             windows=captured["windows"], emitted_frames=captured["emit"],
             gflop_arithmetic=dict(overlap=gflop(captured["windows"], "overlap"), needed_rows=gflop(captured["windows"], "rows"),
                                   needed_rows_in_128_row_tiles=gflop(captured["windows"], "tiles")))
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
out = dict(card=smi, N=N, eos_bias=bias, calibration=tried,
           audio_s_per_wall_s={f"{a}_{r}": statistics.median(v) for (a, r), v in res.items()},
           runs={f"{a}_{r}": v for (a, r), v in res.items()},
           time_to_first_audio_ms={f"{a}_{r}": dict(from_call=stats(fc), from_admission=stats(fa)) for (a, r), (fc, fa) in ttfa.items()},
           codec_per_boundary=codec)
print(json.dumps(out), flush=True)
out_dir = os.environ.get("PTTS_TOOLS_OUT", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools_out"))
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "continuous_stream_time.json"), "w") as f:
    json.dump(out, f, indent=1)
