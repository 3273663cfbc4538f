"""ParlerTTSStreamer: the reference's streaming contract (parler_tts/streamer.py:11-146) over the CUDA codec path.

Contract kept (what `generate(streamer=...)` and consumer threads rely on): `put(value)` receives the initial [B*K, n0] ids (the
BOS column, or the delayed input of a continuation from `decoder_input_ids`) and
then one [B*K] token column per decode step (CPU tensors, as `_sample` hands them over), `end()` closes the stream, and the
object is an iterator over numpy audio chunks fed through a queue (a `timeout` guards both sides).

Two modes:
  * `incremental=False` -- the reference's behaviour: every `play_steps` columns the WHOLE token history is de-delayed and
    decoded again, the part not yet played minus `stride` samples of provisional tail is emitted (O(T^2) codec work, batch 1
    only, parler_tts/streamer.py:66-122).
  * `incremental=True` (SURVEY section 8f rank 1; not in the reference) -- code frames are assembled as their last codebook
    arrives (frame f of codebook k is raw column f + k + 1: no mask is rebuilt over the history), only the NEW frames plus the
    decoder's receptive field (+-10 frames, incremental.py) are decoded, every emitted sample is final, and any batch size works:
    chunks are [B, n] arrays (1-D for B = 1 like the reference); an utterance that has produced a special token (EOS / pad) is
    silent from that frame on.
"""
from __future__ import annotations
import math
from queue import Queue
from typing import Optional

import numpy as np
import torch

from .incremental import IncrementalDecoder, dac_dependency_radius
from .modeling import apply_delay_pattern_mask, build_delay_pattern_mask


class _FrameAssembler:
    """Token columns in, complete code frames out.  Column c (c >= 1) of row b*K + k carries frame c - 1 - k of codebook k
    (the delay pattern, modeling_parler_tts.py:214-276, quirk Q13), so frame f is complete once column f + K has arrived."""

    def __init__(self, num_codebooks: int, codebook_size: int):
        self.K, self.cs = num_codebooks, codebook_size
        self.cols = None          # [B*K, capacity] int64 (CPU)
        self.n = 0                # columns received (the BOS column included)
        self.taken = 0            # frames already handed out
        self.ended = None         # [B] first invalid frame per utterance (or a large number)

    def add(self, value: torch.Tensor):
        v = value.detach().to("cpu", torch.int64)
        v = v if v.dim() == 2 else v[:, None]
        if self.cols is None:
            self.cols = torch.empty(v.shape[0], 256, dtype=torch.int64)
            self.ended = torch.full((v.shape[0] // self.K,), 1 << 40, dtype=torch.int64)
        need = self.n + v.shape[1]
        if need > self.cols.shape[1]:
            grown = torch.empty(self.cols.shape[0], max(need, 2 * self.cols.shape[1]), dtype=torch.int64)
            grown[:, :self.n] = self.cols[:, :self.n]
            self.cols = grown
        self.cols[:, self.n:need] = v
        self.n = need

    @property
    def batch(self) -> int:
        return 0 if self.cols is None else self.cols.shape[0] // self.K

    def complete_frames(self) -> int:
        return max(0, self.n - self.K)

    def take_new(self):
        """Frames completed since the last call: (codes [B, K, n] with special ids replaced by 0, valid [B, n] bool)."""
        lo, hi = self.taken, self.complete_frames()
        if hi <= lo:
            return None, None
        B, K = self.batch, self.K
        rows = self.cols.view(B, K, -1)
        codes = torch.stack([rows[:, k, lo + k + 1:hi + k + 1] for k in range(K)], dim=1)      # [B, K, n]
        bad = (codes >= self.cs).any(dim=1)                                                     # [B, n]
        idx = torch.arange(lo, hi)[None, :].expand(B, -1)
        first_bad = torch.where(bad, idx, torch.full_like(idx, 1 << 40)).min(dim=1).values
        self.ended = torch.minimum(self.ended, first_bad)
        valid = idx < self.ended[:, None]
        self.taken = hi
        return codes.clamp_(max=self.cs - 1).masked_fill_(~valid[:, None, :].expand(-1, K, -1), 0), valid


class ParlerTTSStreamer:
    def __init__(self, model, device: Optional[str] = None, play_steps: Optional[int] = 10, stride: Optional[int] = None,
                 timeout: Optional[float] = None, incremental: bool = False):
        self.decoder = model.decoder
        self.audio_encoder = model.audio_encoder
        self.generation_config = model.generation_config
        self.device = device if device is not None else model.device
        self.audio_kwargs = {"audio_scales": [None]} if model.use_audio_scales else {}
        self.play_steps = int(play_steps)
        cfg = self.audio_encoder.config
        self.hop = math.prod(int(r) for r in cfg.decoder_rates)
        if stride is None:  # the reference's default: a sixth of the samples one `play_steps` window adds (streamer.py:58-60)
            stride = math.floor(cfg.sampling_rate / cfg.frame_rate) * (self.play_steps - self.decoder.num_codebooks) // 6
        self.stride = stride
        self.timeout = timeout
        self.audio_queue: Queue = Queue()
        self.stop_signal = None
        self.incremental = bool(incremental)
        self._frames = _FrameAssembler(self.decoder.num_codebooks, cfg.codebook_size)
        self._history = None      # reference mode: [K, n] token history of the single utterance (device)
        self.to_yield = 0         # reference mode: samples already emitted
        self._inc: Optional[IncrementalDecoder] = None
        self._inc_valid = None    # incremental mode: validity of the frames pushed but not yet emitted

    # -- codec ---------------------------------------------------------------------------------------
    def _decode(self, codes_bkt: torch.Tensor) -> torch.Tensor:
        """codes [B, K, T] -> audio [B, hop * T] on the CUDA DAC path."""
        a = self.audio_encoder.decode(audio_codes=codes_bkt.to(self.device)[None, ...], **({"audio_scales": [None] * codes_bkt.shape[0]} if self.audio_kwargs else {}))
        return a.audio_values[:, 0]

    # -- reference mode: decode the whole history again, keep the unplayed part minus `stride` -----
    def apply_delay_pattern_mask(self, input_ids: torch.Tensor) -> np.ndarray:
        """Same name and result as the reference method (streamer.py:66-94): raw token history [K, n] -> waveform of every
        complete, special-token-free frame."""
        gc = self.generation_config
        ids = input_ids.to(self.device)
        K = self.decoder.num_codebooks
        _, mask = build_delay_pattern_mask(ids[:, :1], gc.bos_token_id, gc.decoder_start_token_id, ids.shape[-1], K)
        ids = apply_delay_pattern_mask(ids, mask)
        free = (mask != gc.bos_token_id) & (mask != gc.pad_token_id)
        codes = ids[free].reshape(1, K, -1)
        ok = (codes >= self.audio_encoder.config.codebook_size).sum(dim=(0, 1)) == 0
        codes = codes[:, :, ok]
        if codes.shape[-1] == 0:
            return np.zeros(0, dtype=np.float32)
        return self._decode(codes)[0].float().cpu().numpy()

    def _flush_reference(self, final: bool):
        if self._frames.cols is None:
            self.on_finalized_audio(np.zeros(self.to_yield), stream_end=final)
            return
        audio = self.apply_delay_pattern_mask(self._frames.cols[:, :self._frames.n])
        if final:
            self.on_finalized_audio(audio[self.to_yield:], stream_end=True)
        else:
            self.on_finalized_audio(audio[self.to_yield: -self.stride])
            self.to_yield += len(audio) - self.to_yield - self.stride

    # -- incremental mode: new frames + receptive-field context only, any batch size -------------------
    def _flush_incremental(self, final: bool):
        if self._inc is None:
            self._inc = IncrementalDecoder(self._decode, self.hop, dac_dependency_radius(self.audio_encoder.config.decoder_rates))
        chunks = []
        codes, valid = self._frames.take_new()
        if codes is not None and codes.shape[0] == 1:   # one utterance: frames holding a special token are dropped, as the
            keep = valid[0]                              # reference (and generate()) do; a batch stays rectangular instead
            codes, valid = codes[..., keep], valid[..., keep]
            if codes.shape[-1] == 0:
                codes = None
        if codes is not None:
            self._inc_valid = valid if self._inc_valid is None else torch.cat([self._inc_valid, valid], dim=1)
            out = self._inc.push(codes)
            if out is not None:
                chunks.append(out)
        if final:
            out = self._inc.finish()
            if out is not None:
                chunks.append(out)
        if chunks:
            audio = torch.cat(chunks, dim=-1).float()
            n = audio.shape[-1] // self.hop                       # frames these samples belong to (emitted in order)
            keep = self._inc_valid[:, :n].to(audio.device).repeat_interleave(self.hop, dim=1)
            self._inc_valid = self._inc_valid[:, n:]
            audio = (audio * keep).cpu().numpy()                   # an utterance is silent after its first special token
        else:
            audio = np.zeros((max(1, self._frames.batch), 0), dtype=np.float32)
        self.on_finalized_audio(audio[0] if audio.shape[0] == 1 else audio, stream_end=final)

    # -- the streaming contract ----------------------------------------------------------------------
    def put(self, value: torch.Tensor):
        if not self.incremental and value.shape[0] // self.decoder.num_codebooks > 1:
            raise ValueError("ParlerTTSStreamer only supports batch size 1")   # (reference :110-112; incremental=True lifts it)
        self._frames.add(value)
        if self.incremental and value.dim() == 2 and value.shape[1] > 1:
            self._flush_incremental(False)   # a continuation's first put holds the whole delayed input: its frames go out first
        elif self._frames.n % self.play_steps == 0:
            (self._flush_incremental if self.incremental else self._flush_reference)(False)

    def end(self):
        (self._flush_incremental if self.incremental else self._flush_reference)(True)

    def on_finalized_audio(self, audio: np.ndarray, stream_end: bool = False):
        self.audio_queue.put(audio, timeout=self.timeout)
        if stream_end:
            self.audio_queue.put(self.stop_signal, timeout=self.timeout)

    def __iter__(self):
        return self

    def __next__(self):
        item = self.audio_queue.get(timeout=self.timeout)
        if item is self.stop_signal:
            raise StopIteration()
        return item
