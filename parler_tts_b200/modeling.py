"""Host-side mirror of the reference's generation surface, calling the sm_90a kernels through the C ABI.

Mirrors (same names, argument meaning and error behaviour; nothing here computes on the CPU):
  build_delay_pattern_mask / apply_delay_pattern_mask   parler_tts/modeling_parler_tts.py:205-276
  ParlerTTSLogitsProcessor                              parler_tts/logits_processors.py:6-53
  ParlerTTSForCausalLM (step operator)                  parler_tts/modeling_parler_tts.py:1824-1974
  ParlerTTSForConditionalGeneration.generate            parler_tts/modeling_parler_tts.py:3322-3653
PyTorch is used for device memory, streams and the one-off side inputs the path does not replace
(text encoder, prompt embedding lookup: SURVEY.md section 1).
"""
from __future__ import annotations
import collections
import contextlib
import ctypes as C
import functools
import json
import math
import os
from typing import Any, NamedTuple, Optional

import numpy as np
import torch

from . import _lib
from .configuration import DACConfig, GenerationConfig, ParlerTTSConfig, ParlerTTSDecoderConfig
from .dac_wrapper import DACModel
from .incremental import dac_dependency_radius

_ACT = {"gelu": 0, "relu": 1, "silu": 2, "swish": 2, "gelu_new": 3, "gelu_pytorch_tanh": 3}


# ---- delay pattern (stand-alone operators) -------------------------------------------------------
def build_delay_pattern_mask(input_ids: torch.LongTensor, bos_token_id: int, pad_token_id: int, max_length: int,
                             num_codebooks: int):
    """Same contract as the reference function: returns (input_ids[:, :first_start], pattern_mask)."""
    ids = input_ids.reshape(-1, num_codebooks, input_ids.shape[-1])
    bsz, K, seq_len = ids.shape
    ids2 = ids.reshape(bsz * K, seq_len).to(torch.int64).contiguous()
    mask = torch.empty(bsz * K, max_length, dtype=torch.int64, device=ids2.device)
    _lib.check(_lib.lib().ptts_delay_build(_lib.ptr(ids2), bsz * K, seq_len, K, int(bos_token_id), int(pad_token_id),
                                           int(max_length), _lib.ptr(mask), _lib.stream_ptr()))
    if max_length < 2 * K - 1:
        return ids2, mask
    first = mask.view(bsz, K, max_length)[:, 0, :]
    starts = (first == -1).nonzero()[:, 1]
    first_start = int(starts.min()) if len(starts) > 0 else seq_len
    out_ids = mask.view(bsz, K, max_length)[..., :first_start].reshape(bsz * K, -1)
    return out_ids, mask


def apply_delay_pattern_mask(input_ids: torch.LongTensor, decoder_pad_token_mask: torch.LongTensor):
    seq_len = input_ids.shape[-1]
    ids = input_ids.reshape(-1, seq_len).to(torch.int64).contiguous()
    mask = decoder_pad_token_mask.reshape(-1, decoder_pad_token_mask.shape[-1]).to(torch.int64).contiguous()
    if mask.shape[-1] < seq_len:
        raise ValueError(f"delay pattern mask is shorter ({mask.shape[-1]}) than the ids ({seq_len})")
    out = torch.empty_like(ids)
    _lib.check(_lib.lib().ptts_delay_apply(_lib.ptr(ids), ids.shape[0], seq_len, seq_len, _lib.ptr(mask), mask.shape[-1],
                                           _lib.ptr(out), _lib.stream_ptr()))
    return out.reshape(input_ids.shape)


def prepare_decoder_input_ids(decoder_input_ids, batch_size: int, num_codebooks: int, vocab_size: int, decoder_start_token_id: int,
                              device) -> torch.Tensor:
    """generate()'s `decoder_input_ids` (audio codes to continue from) -> the BOS-led decoder input [B * K, n0] int64 on `device`.

    Anything `reshape(-1, K, N)` accepts is taken: [B * K, N], [B, K, N] or [1, B, K, N] (generate(return_codes=True)'s audio_codes
    with its frame dimension).  A BOS column is prepended unless every row already starts with it (:3012-3024).  Ids must lie in
    [0, vocab_size] (the embedding tables have vocab_size + 1 rows, :1353)."""
    B, K, V = int(batch_size), int(num_codebooks), int(vocab_size)
    ids = torch.as_tensor(decoder_input_ids)
    if ids.is_floating_point() or ids.is_complex() or ids.dtype == torch.bool:
        raise ValueError(f"decoder_input_ids must hold integer audio codes, got {ids.dtype}")
    N = ids.shape[-1] if ids.dim() >= 1 else 0
    if N < 1 or ids.numel() != B * K * N:
        raise ValueError(f"decoder_input_ids must have batch_size * num_codebooks = {B * K} rows of codes, got shape {tuple(ids.shape)}")
    ids = ids.reshape(B * K, N).to(device=device, dtype=torch.int64)
    lo, hi = int(ids.min()), int(ids.max())
    if lo < 0 or hi > V:
        raise ValueError(f"decoder_input_ids must lie in [0, vocab_size = {V}], got values in [{lo}, {hi}]")
    if bool((ids[:, 0] != decoder_start_token_id).all()):
        ids = torch.cat([torch.full((B * K, 1), int(decoder_start_token_id), dtype=torch.int64, device=ids.device), ids], dim=1)
    return ids.contiguous()


def prepare_ragged_decoder_input_ids(decoder_input_ids, decoder_attention_mask, batch_size: int, num_codebooks: int, vocab_size: int,
                                     decoder_start_token_id: int, device) -> tuple[torch.Tensor, torch.Tensor]:
    """generate()'s `decoder_input_ids` with a `decoder_attention_mask` [B, N] (code prefixes of different lengths) -> (the
    BOS-led decoder input [B * K, n0] int64 on `device`, input_lens [B] int32 on `device`: row b's own columns n0_b, BOS included).

    The mask must be right padding (ones, then zeros); row b's prefix is its first m_b frames, 0 <= m_b <= N, and the ids past it
    are never read.  The BOS column is prepended as prepare_decoder_input_ids does, deciding on the rows that have frames (all
    rows when none has), and a one goes in front of the mask with it (:3025-3031): n0_b = m_b + 1, so a row with m_b = 0 is the
    BOS column alone.  Without the prepended column every row needs m_b >= 1.  n0 = max n0_b; ids in the valid region must lie
    in [0, vocab_size]."""
    B, K, V = int(batch_size), int(num_codebooks), int(vocab_size)
    ids = torch.as_tensor(decoder_input_ids)
    if ids.is_floating_point() or ids.is_complex() or ids.dtype == torch.bool:
        raise ValueError(f"decoder_input_ids must hold integer audio codes, got {ids.dtype}")
    N = ids.shape[-1] if ids.dim() >= 1 else 0
    if N < 1 or ids.numel() != B * K * N:
        raise ValueError(f"decoder_input_ids must have batch_size * num_codebooks = {B * K} rows of codes, got shape {tuple(ids.shape)}")
    m = torch.as_tensor(decoder_attention_mask)
    if m.dim() != 2 or tuple(m.shape) != (B, N):
        raise ValueError(f"decoder_attention_mask must be [batch_size, frames] = [{B}, {N}], got {tuple(m.shape)}")
    m = m.to(device="cpu")
    if m.is_floating_point() or m.is_complex():
        raise ValueError(f"decoder_attention_mask must hold 0 / 1 integers, got {m.dtype}")
    m = m.to(torch.int64)
    if bool(((m != 0) & (m != 1)).any()) or bool((m[:, 1:] > m[:, :-1]).any()):
        raise ValueError("decoder_attention_mask must be right padding: ones, then zeros, in every row")
    frames = m.sum(dim=1)                                                          # m_b
    ids = ids.reshape(B * K, N).to(dtype=torch.int64)
    valid = (torch.arange(N)[None, :] < frames.repeat_interleave(K)[:, None]).to(ids.device)
    if bool(valid.any()):
        lo, hi = int(ids[valid].min()), int(ids[valid].max())
        if lo < 0 or hi > V:
            raise ValueError(f"decoder_input_ids must lie in [0, vocab_size = {V}] inside the mask, got values in [{lo}, {hi}]")
    with_frames = (frames > 0).repeat_interleave(K).to(ids.device)
    prepend = not bool(with_frames.any()) or bool((ids[with_frames, 0] != decoder_start_token_id).all())
    if prepend:
        ids = torch.cat([torch.full((B * K, 1), int(decoder_start_token_id), dtype=torch.int64, device=ids.device), ids], dim=1)
        frames = frames + 1
    elif bool((frames == 0).any()):
        raise ValueError("decoder_attention_mask: a row without frames needs the BOS column, but the codes already start with it "
                         "(pass the rows without their BOS column)")
    n0 = int(frames.max())
    return ids[:, :n0].to(device).contiguous(), frames.to(device=device, dtype=torch.int32)


def ragged_offsets(input_lens: torch.Tensor) -> torch.Tensor:
    """Per-row offsets s_b = n0 - n0_b of a ragged continuation: row b's columns run s_b behind the batch's."""
    return input_lens.max() - input_lens


def check_continuation_length(n0: int, prompt_len: int, max_length: int, max_position_embeddings: int):
    """A continuation from n0 input columns must leave a new column within max_length, and the prompt prefix plus max_length
    positions must fit the position table."""
    if n0 >= max_length:
        raise ValueError(f"decoder_input_ids has {n0} columns (BOS included): max_length {max_length} leaves no new token; "
                         "raise max_length or pass max_new_tokens")
    if prompt_len + max_length > max_position_embeddings:
        raise ValueError(f"{prompt_len} prompt positions + max_length {max_length} exceed max_position_embeddings {max_position_embeddings}")


def resolve_num_return_sequences(gc) -> int:
    """generate()'s takes per description, validated as transformers does (GenerationConfig.validate): an int >= 1, and > 1 only
    with sampling."""
    n = gc.num_return_sequences
    if isinstance(n, bool) or not isinstance(n, int) or n < 1:
        raise ValueError(f"`num_return_sequences` has to be a strictly positive integer, got {n!r}")
    if n > 1 and not gc.do_sample:
        raise ValueError(f"Greedy methods without beam search do not support `num_return_sequences` different than 1 (got {n}).")
    return n


def expand_takes(ids: torch.Tensor, batch_size: int, num_codebooks: int, takes: int) -> torch.Tensor:
    """[B * K, n] utterance-major code rows -> [B * takes * K, n]: the K rows of utterance b, as one group, once for each of its
    takes, so that take j of utterance b is utterance b * takes + j (never a repeat of single [B * K] rows)."""
    return ids.reshape(batch_size, num_codebooks, -1).repeat_interleave(takes, dim=0).reshape(batch_size * takes * num_codebooks, -1)


def check_ragged_generate(streamer, logits_processor, stopping_criteria, gc):
    """What generate() refuses with code prefixes of different lengths (a decoder_attention_mask or a list of input_values): the
    streamer and the caller's processors / criteria (the host-driven loop hands them one rectangular input_ids),
    output_attentions / output_hidden_states / return_token_timestamps (their probes take one position for the batch), and
    min_length without min_new_tokens (it counts each row's own prefix, which one min_new_tokens for the batch cannot)."""
    bad = []
    if streamer is not None:
        bad.append("streamer")
    if logits_processor:
        bad.append("logits_processor")
    if stopping_criteria:
        bad.append("stopping_criteria")
    for k in ("output_attentions", "output_hidden_states", "return_token_timestamps"):
        if getattr(gc, k, False):
            bad.append(k)
    if gc.min_new_tokens is None and (getattr(gc, "min_length", 0) or 0) > 0:
        bad.append("min_length (pass min_new_tokens)")
    if bad:
        raise ValueError(f"code prefixes of different lengths (decoder_attention_mask, or a list of input_values) do not support "
                         f"{', '.join(bad)}")


def take_shards(batch_size: int, takes: int, limit: Optional[int]) -> list[tuple[int, int, int, int]]:
    """The sessions generate() runs for batch_size descriptions x `takes` takes: (first description, end, first output row, end)
    each, every session's rows whole groups of takes of its descriptions (its takes = rows / descriptions).  limit: the rows one
    session may hold (None: one session).  takes <= limit: floor(limit / takes) descriptions per session; takes > limit: up to
    `limit` takes of one description per session."""
    n = batch_size * takes
    if limit is None or n <= limit:
        return [(0, batch_size, 0, n)]
    if takes <= limit:
        g = limit // takes
        return [(d0, min(batch_size, d0 + g), d0 * takes, min(batch_size, d0 + g) * takes) for d0 in range(0, batch_size, g)]
    return [(b, b + 1, b * takes + j0, b * takes + min(takes, j0 + limit)) for b in range(batch_size) for j0 in range(0, takes, limit)]


def compact_valid_frames(codes: torch.Tensor, codebook_size: int) -> tuple[torch.Tensor, torch.Tensor]:
    """codes [B, K, T] -> (codes with each row's valid frames moved to the front in order, valid count [B] int64).

    A frame is valid when all K of its ids are < codebook_size: the frames the reference's per-sample branch keeps with its
    boolean gather (:3631-3633).  Invalid frames can sit mid-row (untrained weights, quirk Q5), so this is a stable sort of
    the frame order by validity; what lies past a row's count is left over and never decoded."""
    valid = (codes < codebook_size).all(dim=1)                                       # [B, T]
    order = torch.sort((~valid).to(torch.uint8), dim=1, stable=True).indices          # valid frames first, in order
    packed = torch.gather(codes, 2, order[:, None, :].expand_as(codes))
    return packed, valid.sum(dim=1)


def codes_to_waveform(audio_encoder: DACModel, codes: torch.Tensor, codebook_size: int, dtype: torch.dtype):
    """generate()'s codes -> waveform step for codes [B, K, T] that may hold ids >= codebook_size (EOS / pad after an
    utterance's end): each row decodes its valid frames alone (:3615-3641), here in one ragged codec call.

    Returns (audio [B, hop * max n_b] zero-padded after each row, lengths: hop * n_b, or 1 for a row without a valid frame).
    A batch with no valid frame at all gives [B, 1] zeros in `dtype`, like the reference's pad_sequence of 1-sample rows."""
    packed, n = compact_valid_frames(codes, codebook_size)
    return packed_to_waveform(audio_encoder, packed, n.tolist(), dtype)


def packed_to_waveform(audio_encoder: DACModel, packed: torch.Tensor, n_host: list[int], dtype: torch.dtype):
    """codes_to_waveform after the compaction: packed [B, K, T] with row b's n_host[b] valid frames first."""
    B = packed.shape[0]
    T = max(n_host, default=0)
    if T == 0:
        return torch.zeros(B, 1, device=packed.device, dtype=dtype), [1] * B
    audio = audio_encoder.decode(audio_codes=packed[None, :, :, :T], audio_scales=[None] * B, frame_lengths=n_host).audio_values
    hop = audio_encoder.hop_length
    return audio.squeeze(1), [hop * v if v > 0 else 1 for v in n_host]


# ---- continuous batching (generate_continuous) --------------------------------------------------------------------------------
def check_continuous_generate(gc, mk: dict, streamer=None, logits_processor=None, stopping_criteria=None):
    """What generate_continuous() refuses: whatever counts from one batch column for all rows (forced_eos_token_id,
    exponential_decay_length_penalty, begin_suppress_tokens), the per-step outputs and probes (output_scores, output_logits,
    output_attentions, output_hidden_states, return_token_timestamps), a streamer, the caller's processors and criteria (the
    host-driven loop), continuations (decoder_input_ids, decoder_attention_mask, input_values) and num_return_sequences > 1."""
    bad = []
    if streamer is not None:
        bad.append("streamer")
    if logits_processor:
        bad.append("logits_processor")
    if stopping_criteria:
        bad.append("stopping_criteria")
    for k in ("decoder_input_ids", "decoder_attention_mask", "input_values"):
        if mk.get(k) is not None:
            bad.append(k)
    for k in ("output_scores", "output_logits", "output_attentions", "output_hidden_states", "return_token_timestamps"):
        if getattr(gc, k, False):
            bad.append(k)
    for k in ("forced_eos_token_id", "exponential_decay_length_penalty", "begin_suppress_tokens"):
        if getattr(gc, k, None) is not None:
            bad.append(k)
    if gc.num_return_sequences != 1:
        bad.append("num_return_sequences > 1")
    if bad:
        raise ValueError(f"generate_continuous() does not support {', '.join(bad)}")


def check_continuous_counts(stream, batch_size, refill_every):
    """generate_continuous()'s and continuous_engine()'s first checks, before anything touches the model."""
    if not isinstance(stream, bool):
        raise ValueError(f"stream must be a bool, got {stream!r}")
    if isinstance(batch_size, bool) or not isinstance(batch_size, int) or batch_size < 1:
        raise ValueError(f"batch_size must be a positive int, got {batch_size!r}")
    if isinstance(refill_every, bool) or not isinstance(refill_every, int) or refill_every < 1:
        raise ValueError(f"refill_every must be a positive int, got {refill_every!r}")


def continuous_settings(model, kwargs: dict, streamer, logits_processor, stopping_criteria):
    """generate_continuous()'s and continuous_engine()'s generation settings -> (config, model kwargs, max_length in each
    request's own columns, suppress_special), with the device loop's and check_continuous_generate's rejections."""
    import copy
    gc = copy.deepcopy(model.generation_config)
    suppress_special = kwargs.pop("_suppress_special", False)
    user_max_length = kwargs.get("max_length")
    mk = gc.update(**kwargs)
    unknown = sorted(k for k in mk if k not in model._MODEL_KWARGS)
    if unknown:
        raise ValueError(f"The following `model_kwargs` are not used by the model: {unknown}")
    unsupported = {k: getattr(gc, k) for k, neutral in model._NEUTRAL_GENERATION_KNOBS.items() if getattr(gc, k, neutral) != neutral}
    if unsupported or gc.num_beams != 1:
        raise ValueError(f"generation options {unsupported or {'num_beams': gc.num_beams}} are not supported by the device loop")
    for k in ("output_attentions", "output_hidden_states"):   # model kwargs in generate(); here refused like the config fields
        if mk.get(k):
            setattr(gc, k, True)
    check_continuous_generate(gc, mk, streamer, logits_processor, stopping_criteria)
    if gc.max_new_tokens is not None:
        max_length = int(gc.max_new_tokens) + 1
    else:
        max_length = int(user_max_length if user_max_length is not None else gc.max_length)
    if max_length < 2:
        raise ValueError(f"max_length must allow at least one new token, got {max_length}")
    return gc, mk, max_length, suppress_special


def slot_outputs(raw: torch.Tensor, eos_last: torch.Tensor, cur_len, shift: torch.Tensor, max_length, codebook_size: int,
                 live: bool = False):
    """Every slot's state at a refill boundary, on the device (nothing here waits for it).  raw [B, K, ld] the history, eos_last [B]
    = 1 + the column of the last codebook's first EOS (0: none; a row stopped by max_length records the PAD it writes after, when
    pad == eos: hence the clamp), cur_len and shift [B] the slot columns.  Returns (finished [B], frames F [B], codes [B, K,
    max_length] with the F de-delayed frames first, the same with the valid frames compacted to the front as codes_to_waveform
    does, and their count [B]).  A request that ended with n history columns gets generate()'s cut (_codes_from_raw over its own columns): frame f
    of codebook k is column f + k + 1, F = n - K, once n reaches the delay pattern's 2K - 1 columns; below that every column, F = n.
    live: an unfinished slot with col = cur_len - shift columns also gets its complete frames, F = col - K (the last codebook of
    frame f is column f + K), and none while col < 2K - 1, where the row may still end under the cut without the pattern.  Its
    compacted frames are then a prefix of those its finished cut will hold (the compaction keeps the frame order).
    max_length: an int, or an integer tensor [B] of per-slot limits (ContinuousEngine's per-request max_new_tokens): slot b is then
    cut at its own max_length[b], as generate() with that max_length cuts it, and codes / packed are ld frames wide."""
    B, K, ld = raw.shape
    if isinstance(max_length, torch.Tensor):
        L, width = max_length.to(device=eos_last.device, dtype=eos_last.dtype), ld
        n = torch.where(eos_last > 0, torch.minimum(eos_last, L), L)
    else:
        L = width = int(max_length)
        n = torch.where(eos_last > 0, eos_last.clamp(max=L), torch.full_like(eos_last, L))
    finished = (eos_last > 0) | (cur_len - shift >= L)
    pattern = n >= 2 * K - 1
    frames = torch.where(pattern, n - K, n)
    if live:
        col = cur_len - shift
        pattern = pattern | ~finished
        frames = torch.where(finished, frames, torch.where(col >= 2 * K - 1, col - K, torch.zeros_like(col)).to(frames.dtype))
    f = torch.arange(width, device=raw.device)
    off = pattern[:, None].long() * torch.arange(1, K + 1, device=raw.device)[None, :]
    codes = torch.gather(raw, 2, (f[None, None, :] + off[:, :, None]).clamp(max=ld - 1))
    valid = (codes < codebook_size).all(dim=1) & (f[None, :] < frames[:, None])
    order = torch.sort((~valid).to(torch.uint8), dim=1, stable=True).indices
    packed = torch.gather(codes, 2, order[:, None, :].expand_as(codes))
    return finished, frames, codes, packed, valid.sum(dim=1)


def stream_windows(n_valid: list, emitted: list, finishing: list, radius: int) -> list[tuple[int, int, int, int]]:
    """A streamed boundary's codec windows, one (start, n, lo, hi) per slot: decode valid frames [start, start + n) and emit the
    samples of window frames [lo, hi), i.e. of frames [start + lo, start + hi).  n_valid: each slot's valid frames so far,
    emitted: the frames already played (None: no request in the slot), finishing: the slot's request ends at this boundary.
    Frame f's samples depend on frames [f - radius, f + radius] (incremental.dac_dependency_radius), so a live slot emits up
    to n_valid - radius, once that passes `emitted`, from a window that starts radius frames before `emitted` (or at frame 0).
    A finishing slot emits up to n_valid: its end is the true end, which the decode's zero padding stands for.  Every other slot
    gets n = 0."""
    out = []
    for n, e, fin in zip(n_valid, emitted, finishing):
        upto = n if fin else n - radius
        if e is None or not (fin or upto > e):
            out.append((0, 0, 0, 0))
            continue
        start = max(0, e - radius)
        out.append((start, n - start, e - start, upto - start))
    return out


def refill_rows(t: Optional[torch.Tensor], first: int, count: int, rows: int) -> Optional[torch.Tensor]:
    """Rows [first, first + count) of a per-request input, padded to `rows` rows by repeating the last one: a refill prefills a
    session of batch_size rows, so its GEMMs take the kernels a batch_size-row generate() shard takes (the padding rows are never
    imported)."""
    if t is None:
        return None
    last = t[first + count - 1:first + count]
    return torch.cat([t[first:first + count], last.expand(rows - count, *t.shape[1:])])


def rebase_slots(cur_len: int, cols: list) -> tuple[int, list[int]]:
    """A refill boundary's new batch column and row offsets.  cols[b]: the column slot b draws next, None for an idle slot.  The
    batch column becomes the largest live column, one more when that keeps cur_len's parity (the ParlerTTSLogitsProcessor state
    is double-buffered on it), and row b's offset is cur_len - cols[b] >= 0; idle slots are parked at column 1."""
    top = max((c for c in cols if c is not None), default=1)
    new = top + ((top - cur_len) & 1)
    return new, [new - (1 if c is None else c) for c in cols]


class ContinuousRun:
    """generate_continuous()'s iterator of (request index, waveform[, codes]) in completion order, or with stream=True of
    (request index, chunk, final[, codes]) events.  `refills` logs every request
    put into a slot at a boundary as (slot, request, batch column of that boundary); `boundaries` and `steps` count the
    boundaries and the decode steps enqueued (those of the ContinuousEngine it drains)."""

    def __init__(self, engine: "ContinuousEngine"):
        self.engine = engine
        self._it = engine._drain()

    refills = property(lambda self: self.engine.refills)
    boundaries = property(lambda self: self.engine.boundaries)
    steps = property(lambda self: self.engine.steps)

    def __iter__(self):
        return self

    def __next__(self):
        return next(self._it)


def left_pad(states: Optional[torch.Tensor], mask: Optional[torch.Tensor], n: int, what: str):
    """One request's states [1, s, H] and mask [1, s] (None: every position attended) left-padded to n positions with zero states
    and a zero mask, the way a padded batch holds a shorter description or prompt.  No padding keeps the mask as given.  Raises
    ValueError for s > n."""
    if states is None:
        return None, None
    s = states.shape[1]
    if s > n:
        raise ValueError(f"the {what} has {s} positions, more than the engine's max_{what}_length = {n}")
    if s == n:
        return states, mask
    m = torch.ones(1, s, dtype=torch.long, device=states.device) if mask is None else mask.to(states.device, torch.long)
    pad = n - s
    states = torch.cat([states.new_zeros(1, pad, states.shape[2]), states], dim=1)
    return states, torch.cat([m.new_zeros(1, pad), m], dim=1)


class ContinuousEngine:
    """Online continuous batching (ParlerTTSForConditionalGeneration.continuous_engine): requests are submitted, cancelled and
    stepped while the batch decodes.  One live session of `batch_size` slots; every step() reads the boundary of the interval the
    previous step() launched, yields its events, admits queued requests into the free slots and launches the next `refill_every`
    decode steps before it returns, so the device decodes while the caller handles the events and submits.

    Request r draws with Philox key r (its submission index), what row r of one generate() over the submissions in order draws; its
    codes and waveform equal that row's under the conditions generate_continuous() states.  Each request may have its own
    max_new_tokens in [2K - 2, the engine's bound] (K codebooks): the slot sampler stops it and applies its delay pattern at its
    own limit (ptts_generate_set_slots2), and its cut follows that limit (slot_outputs with per-slot limits).

    Calls are serialised by the caller (one handle is not thread-safe): submit() and cancel() belong between step() calls."""

    QUEUED, LIVE, DONE, CANCELLED = range(4)

    def __init__(self, model, sampling: "Sampling", batch_size: int, refill_every: int, S: int, P: int, stream: bool,
                 return_codes: bool):
        self._m, self._s = model, sampling
        self.batch_size, self.refill_every, self.S, self.P = batch_size, refill_every, S, P
        self.stream, self.return_codes = stream, return_codes
        self.max_length = sampling.max_length
        self._K, self._cs = model.config.decoder.num_codebooks, model.config.audio_encoder.codebook_size
        self._radius = dac_dependency_radius(model.audio_encoder.config.decoder_rates)
        L, B = self.max_length, batch_size
        self._live = self._fill = None   # the live and the refill session, made at the first admission and the first refill
        self._reqs: list = []       # per request: (enc, enc mask, prompt, prompt mask, max_length) until admitted, then None
        self._status: list[int] = []
        self._queue: collections.deque = collections.deque()
        self._slot_req: list = [None] * B
        self._slot_len = [L] * B    # each slot's max_length (idle slots: the bound)
        self._cols = [1] * B        # the column each slot draws next
        self._shift = [0] * B
        self._emitted = [0] * B     # stream: valid frames of each slot's request already played
        self._cur_len = 2
        self._running = False       # an interval is in flight whose boundary has not been read
        self.refills: list[tuple[int, int, int]] = []
        self.boundaries = self.steps = 0

    # -- requests -------------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def submit(self, input_ids=None, attention_mask=None, prompt_input_ids=None, prompt_attention_mask=None, encoder_outputs=None,
               max_new_tokens=None, prompt_hidden_states=None) -> int:
        """Queue one request (batch of 1: a description, or `encoder_outputs`, and the prompt) and return its id, its submission
        index.  Its conditioning runs now (text encoder, enc_to_dec_proj, the prompt_cross_attention assembly); the description
        states are left-padded to max_description_length and the prompt to max_prompt_length.  No decode work is launched: the
        request is admitted at a later step().  max_new_tokens: None (the engine's bound) or an int in [2K - 2, the bound]."""
        limit = self._limit(max_new_tokens)
        enc, em, ph, pm, _, _ = self._m._conditioning("submit", input_ids, attention_mask, encoder_outputs, prompt_input_ids,
                                                      prompt_attention_mask, prompt_hidden_states,
                                                      cross_prompt_after_encoder_outputs=True)
        if enc.shape[0] != 1 or (ph is not None and ph.shape[0] != 1):
            raise ValueError(f"submit() takes one request, got a batch of {enc.shape[0]}")
        return self._submit(enc, em, ph, pm, limit)

    def _limit(self, max_new_tokens) -> int:
        if max_new_tokens is None:
            return self.max_length
        if isinstance(max_new_tokens, bool) or not isinstance(max_new_tokens, int):
            raise ValueError(f"max_new_tokens must be an int, got {max_new_tokens!r}")
        lo = max(2 * self._K - 1, 2)
        if self.max_length < lo:
            raise ValueError(f"an engine with max_length {self.max_length} < {lo} (below the delay pattern's 2K - 1 columns) "
                             "takes no per-request max_new_tokens")
        if not lo - 1 <= max_new_tokens <= self.max_length - 1:
            raise ValueError(f"max_new_tokens {max_new_tokens} outside [{lo - 1}, {self.max_length - 1}] (2K - 2 .. the engine's bound)")
        return max_new_tokens + 1

    def _submit(self, enc, em, ph, pm, limit: int) -> int:
        if ph is not None and self.P == 0:
            raise ValueError("a prompt on an engine with max_prompt_length = 0")
        if ph is None and self.P > 0:
            raise ValueError(f"every request on an engine with max_prompt_length = {self.P} needs a prompt")
        enc, em = left_pad(enc, em, self.S, "description")
        ph, pm = left_pad(ph, pm, self.P, "prompt")
        rid = len(self._reqs)
        self._reqs.append((enc, em, ph, pm, limit))
        self._status.append(self.QUEUED)
        self._queue.append(rid)
        return rid

    def cancel(self, rid: int) -> bool:
        """Drop request rid: a queued one at once, a live one at the next boundary (its slot is free then; it yields nothing more and
        takes no codec call).  False if it already finished or was cancelled; ValueError for an id never returned by submit()."""
        if isinstance(rid, bool) or not isinstance(rid, int) or not 0 <= rid < len(self._status):
            raise ValueError(f"no request {rid!r}: ids are 0 .. {len(self._status) - 1}")
        st = self._status[rid]
        if st == self.QUEUED:
            self._queue.remove(rid)
            self._reqs[rid] = None
        elif st != self.LIVE:
            return False
        self._status[rid] = self.CANCELLED
        return True

    @property
    def idle(self) -> bool:
        """No live and no queued request."""
        return not self._queue and all(r is None or self._status[r] == self.CANCELLED for r in self._slot_req)

    # -- the loop -------------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self) -> list:
        """One boundary and one interval: the events of the boundary of the interval the previous step() launched (the tuples
        generate_continuous() yields), after admitting queued requests into the free slots and launching the next refill_every
        decode steps.  An idle engine returns [] and launches nothing."""
        if self.idle:
            return []
        events, done = [], None
        if self._running:
            events, done = self._boundary()
        self._admit()
        self._running = any(r is not None for r in self._slot_req)
        if self._running:
            self._cur_len, self._shift = rebase_slots(self._cur_len, [c if r is not None else None
                                                                      for c, r in zip(self._cols, self._slot_req)])
            lims = None if all(v == self.max_length for v in self._slot_len) else self._slot_len
            self._live.set_slots(self._cur_len, self._shift, [0 if r is None else r for r in self._slot_req], lims)
            self._live.decode_steps(self.refill_every)   # enqueued before the finished requests' codec call and the caller's turn
            self.steps += self.refill_every
        if done is not None and done[0] and not self.stream:
            # the codes were cut before any import overwrote their slots; the codec call queues behind the next interval
            slots, reqs, codes, packed, frames, n_valid = done
            audio, lengths = packed_to_waveform(self._m.audio_encoder, torch.stack([packed[b] for b in slots]),
                                                [n_valid[b] for b in slots], self._m.dtype)
            for j, (b, r) in enumerate(zip(slots, reqs)):
                wav = audio[j, :lengths[j]]
                events.append((r, wav, codes[b, :, :frames[b]]) if self.return_codes else (r, wav))
        return events

    def _boundary(self):
        """Read the boundary in one host sync (every slot's outcome is computed on the device first): free the cancelled and the
        finished slots; with stream=True enqueue the boundary's codec windows.  Returns (stream events, the finished slots)."""
        B, K, live = self.batch_size, self._K, self._live
        self.boundaries += 1
        rows = torch.tensor([self._shift, self._slot_len], dtype=torch.int32).pin_memory().to(self._m.device, non_blocking=True)
        fin, frames, codes, packed, n_valid = slot_outputs(live.raw_ids.view(B, K, -1), live.eos_seen.view(B, K)[:, K - 1],
                                                           live.state[0], rows[0], rows[1], self._cs, live=self.stream)
        status = torch.cat([live.state[:1].long(), fin.long(), frames.long(), n_valid.long()]).cpu().tolist()
        self._cur_len = status[0]
        fin, frames, n_valid = status[1:1 + B], status[1 + B:1 + 2 * B], status[1 + 2 * B:]
        self._cols = [self._cur_len - sh for sh in self._shift]
        for b, r in enumerate(self._slot_req):
            if r is not None and self._status[r] == self.CANCELLED:
                self._slot_req[b] = None
        events = self._stream_events(packed, codes, fin, frames, n_valid) if self.stream else []
        slots = [b for b, r in enumerate(self._slot_req) if r is not None and fin[b]]
        reqs = [self._slot_req[b] for b in slots]
        for b, r in zip(slots, reqs):
            self._status[r] = self.DONE
            self._slot_req[b] = None
        return events, (slots, reqs, codes, packed, frames, n_valid)

    def _admit(self):
        """Queued requests into free slots: the live session's own prefill the first time, then a prefill of the refill session
        and ptts_session_import_rows.  Request r takes row r - r0 of the prefill (r0 the first admitted), so that row_base r0 * K
        gives it Philox key r; rows of no admitted request repeat the last one (one prefill of batch_size rows, whose GEMMs take a
        batch_size-row batch's kernels)."""
        free = [b for b, r in enumerate(self._slot_req) if r is None]
        if not free or not self._queue:
            return
        B, r0, picked = self.batch_size, self._queue[0], []
        while self._queue and len(picked) < len(free) and self._queue[0] - r0 < B:
            picked.append(self._queue.popleft())
        by_row = {r - r0: self._reqs[r] for r in picked}
        last = self._reqs[picked[-1]]
        rows = [by_row.get(j, last) for j in range(B)]
        conds = self._stack(rows)
        s, eng, first = self._s, self._m.decoder.engine, self._live is None
        if first:
            # max_input_len 2 gives the per-row offsets; finished rows decode PAD until their boundary, hence + refill_every
            self._live = GenSession(eng, B, self.P, self.S, self.P + self.max_length + self.refill_every, max_input_len=2)
            sess, slots = self._live, [r - r0 for r in picked]
        else:
            if self._fill is None:
                self._fill = GenSession(eng, B, self.P, self.S, self.P + self.max_length, max_input_len=2)
            sess, slots = self._fill, free[:len(picked)]
        sess.begin(s.max_length, do_sample=s.do_sample, temperature=s.temperature, top_k=s.top_k, top_p=s.top_p,
                   min_new_tokens=s.min_new_tokens, seed=s.seed, suppress_special=s.suppress_special, codebook_size=s.codebook_size,
                   row_base=r0 * self._K, ext=s.ext, lext=s.lext)
        enc, em, ph, pm = conds
        sess.prefill(ph, pm, enc, em)
        sess.sample()   # the first column, drawn under the engine's max_length (set_slots2 states why that is the request's own)
        if not first:
            self._live.import_rows(self._fill, [r - r0 for r in picked], slots)
        for r, b in zip(picked, slots):
            self._slot_req[b], self._cols[b], self._emitted[b], self._slot_len[b] = r, 2, 0, self._reqs[r][4]
            self._status[r], self._reqs[r] = self.LIVE, None
            if not first:
                self.refills.append((b, r, self._cur_len))

    def _stack(self, rows) -> list:
        """The rows' (description states, mask, prompt states, mask) as batch tensors.  A mask is None when no row has one; a row
        without one (a request given no mask, at full length) then attends everywhere."""
        out, dev = [], self._m.device
        for i, n in ((0, None), (1, self.S), (2, None), (3, self.P)):
            ts = [row[i] for row in rows]
            if all(t is None for t in ts):
                out.append(None)
            elif n is None:
                out.append(torch.cat(ts))
            else:
                out.append(torch.cat([torch.ones(1, n, dtype=torch.long, device=dev) if t is None else t.to(dev, torch.long) for t in ts]))
        return out

    def _stream_events(self, packed, codes, fin, frames, n_valid):
        """One streamed boundary: every slot's window through one windowed codec call (enqueued here, waited for by nobody), and
        the events, in slot order.  Advances `_emitted`."""
        m, slot_req, emitted = self._m, self._slot_req, self._emitted
        wins = stream_windows(n_valid, [e if r is not None else None for e, r in zip(emitted, slot_req)],
                              [r is not None and bool(f) for r, f in zip(slot_req, fin)], self._radius)
        # a fresh buffer per boundary: the chunks yielded are views into it
        audio = m.audio_encoder._decode_windows(packed, wins) if any(w[1] > 0 for w in wins) else None
        hop, events = m.audio_encoder.hop_length, []
        for b, (r, (start, n, lo, hi)) in enumerate(zip(slot_req, wins)):
            final = r is not None and bool(fin[b])
            if r is None or not (final or hi > lo):
                continue
            if final and n_valid[b] == 0:      # no valid frame: the [1] zero waveform, as stream=False gives
                chunk = torch.zeros(1, device=m.device, dtype=m.dtype)
            elif hi > lo:
                chunk = audio[b, lo * hop:hi * hop]
                emitted[b] = start + hi
            else:
                chunk = torch.zeros(0, device=m.device, dtype=m.dtype)
            if self.return_codes:
                events.append((r, chunk, final, codes[b, :, :frames[b]] if final else None))
            else:
                events.append((r, chunk, final))
        return events

    def _drain(self):
        """generate_continuous()'s loop: step until idle, yielding the events."""
        while not self.idle:
            yield from self.step()


def shift_tokens_right(input_ids: torch.Tensor, pad_token_id: int, decoder_start_token_id: int):
    """The reference's shift_tokens_right (:308-323): one position to the right along dim 1, decoder_start_token_id first, -100
    replaced by pad_token_id.  Host-side integer work: labels [B, T, K] -> the decoder input [B, T, K]."""
    if decoder_start_token_id is None:
        raise ValueError("Make sure to set the decoder_start_token_id attribute of the model's configuration.")
    if pad_token_id is None:
        raise ValueError("Make sure to set the pad_token_id attribute of the model's configuration.")
    shifted = input_ids.new_zeros(input_ids.shape)
    shifted[:, 1:] = input_ids[:, :-1].clone()
    shifted[:, 0] = decoder_start_token_id
    shifted.masked_fill_(shifted == -100, pad_token_id)
    return shifted


def scoring_label_mask(labels: torch.Tensor, decoder_input_ids: torch.Tensor, bos_token_id: int, eos_token_id: int):
    """The reference's loss mask (:1935-1946): BOS labels become -100, and a cell (b, t, k) counts iff its label is not -100 and its
    decoder input id is not eos.  labels [B, T, K], decoder_input_ids [B * K, T] -> (labels, mask [B, T, K] bool).  ptts_score
    applies the same rule on the device; this mirror is what the tests hold against the reference."""
    B, T, K = labels.shape
    labels = labels.masked_fill(labels == bos_token_id, -100)
    dec = decoder_input_ids.reshape(B, K, T).transpose(1, 2)
    return labels, (dec != eos_token_id) & (labels != -100)


def check_scoring_inputs(labels, decoder_input_ids, decoder_attention_mask, *, batch_size: int, num_codebooks: int, vocab_size: int,
                         pad_token_id: int, decoder_start_token_id: int, prompt_len: int, max_position_embeddings: int):
    """forward()'s decoder side -> (labels [B, T, K] int64 or None, decoder input [B * K, T] int64), on the inputs' device.

    Without decoder_input_ids the input is shift_tokens_right(labels).transpose(1, 2) (:2820-2823).  Raises ValueError for labels
    outside {-100} u [0, vocab_size), decoder ids outside [0, vocab_size], shapes that do not match the batch / codebooks / each
    other, a decoder_attention_mask that is not right padding, and prompt_len + T above max_position_embeddings."""
    B, K, V = int(batch_size), int(num_codebooks), int(vocab_size)

    def integer(t, name):
        t = torch.as_tensor(t)
        if t.is_floating_point() or t.is_complex() or t.dtype == torch.bool:
            raise ValueError(f"{name} must hold integer ids, got {t.dtype}")
        return t.to(torch.int64)

    if labels is None and decoder_input_ids is None:
        raise ValueError("forward() needs `labels` or `decoder_input_ids`")
    if labels is not None:
        labels = integer(labels, "labels")
        if labels.dim() != 3 or labels.shape[0] != B or labels.shape[2] != K or labels.shape[1] < 1:
            raise ValueError(f"labels must be [batch_size = {B}, sequence_length, num_codebooks = {K}], got {tuple(labels.shape)}")
        if not bool(((labels == -100) | ((labels >= 0) & (labels < V))).all()):
            raise ValueError(f"labels must be -100 or lie in [0, vocab_size = {V})")
    if decoder_input_ids is None:
        dec = shift_tokens_right(labels, pad_token_id, decoder_start_token_id).transpose(1, 2)
    else:
        dec = integer(decoder_input_ids, "decoder_input_ids")
        if dec.dim() not in (2, 3) or dec.shape[-1] < 1 or dec.numel() != B * K * dec.shape[-1] or dec.shape[0] not in (B, B * K):
            raise ValueError(f"decoder_input_ids must be [batch_size * num_codebooks = {B * K}, T] or [{B}, {K}, T], got {tuple(dec.shape)}")
        if labels is not None and dec.shape[-1] != labels.shape[1]:
            raise ValueError(f"decoder_input_ids has {dec.shape[-1]} positions, labels {labels.shape[1]}")
        lo, hi = int(dec.min()), int(dec.max())
        if lo < 0 or hi > V:
            raise ValueError(f"decoder_input_ids must lie in [0, vocab_size = {V}], got values in [{lo}, {hi}]")
    dec = dec.reshape(B * K, -1).contiguous()
    T = dec.shape[1]
    if decoder_attention_mask is not None:
        m = torch.as_tensor(decoder_attention_mask)
        if tuple(m.shape) != (B, T):
            raise ValueError(f"decoder_attention_mask must be [{B}, {T}], got {tuple(m.shape)}")
        m = m.to(torch.int64)
        # right padding only: under the causal mask it changes no position the loss keeps, so it is accepted and not needed
        if not bool(((m == 0) | (m == 1)).all()) or not bool((m[:, 1:] <= m[:, :-1]).all()):
            raise ValueError("decoder_attention_mask must be right padding (ones, then zeros)")
    if prompt_len + T > max_position_embeddings:
        raise ValueError(f"{prompt_len} prompt positions + {T} decoder positions exceed max_position_embeddings {max_position_embeddings}")
    return labels, dec


def prompt_cross_states(enc_hidden: torch.Tensor, enc_mask: Optional[torch.Tensor], prompt: torch.Tensor,
                        prompt_mask: Optional[torch.Tensor], embed_prompts: torch.Tensor, positions: torch.Tensor):
    """config.prompt_cross_attention: the transcript prompt as cross-attention keys after the description (reference :3099-3130,
    forward :2791-2811) -> (states [B, S + P, H], mask [B, S + P] or None).

    prompt: ids [B, P] (looked up in embed_prompts) or states [B, P, H]; positions: the [max_position_embeddings, H] sinusoidal
    table.  The prompt becomes prompt + positions[0:P] in the tables' dtype; it is not multiplied by its mask.  If only one of the
    two masks is given, the other becomes ones; with neither there is no mask.  Raises ValueError when P exceeds the table."""
    B, S = enc_hidden.shape[:2]
    P = prompt.shape[1]
    if P > positions.shape[0]:
        raise ValueError(f"the prompt has {P} tokens, more than max_position_embeddings = {positions.shape[0]} positions")
    if prompt.shape[0] != B or prompt.dim() not in (2, 3) or (prompt_mask is not None and tuple(prompt_mask.shape) != (B, P)):
        raise ValueError(f"the prompt must be [{B}, P] ids or [{B}, P, H] states with a [{B}, P] mask, got {tuple(prompt.shape)}"
                         f" and {None if prompt_mask is None else tuple(prompt_mask.shape)}")
    if prompt.dim() == 2:
        prompt = torch.nn.functional.embedding(prompt.to(embed_prompts.device), embed_prompts)
    prompt = prompt.to(device=positions.device, dtype=positions.dtype) + positions[:P]
    if prompt_mask is not None and enc_mask is None:
        enc_mask = torch.ones(B, S, dtype=prompt_mask.dtype, device=prompt_mask.device)
    elif enc_mask is not None and prompt_mask is None:
        prompt_mask = torch.ones(B, P, dtype=enc_mask.dtype, device=enc_mask.device)
    states = torch.cat([enc_hidden.to(prompt.device, prompt.dtype), prompt], dim=1)
    mask = None if prompt_mask is None else torch.cat([enc_mask, prompt_mask.to(enc_mask.device)], dim=1)
    return states, mask


def resolve_sampling_ext(gc, n0: int):
    """The further processors of transformers' `_get_logits_processor` from a GenerationConfig -> (ext, min_new_tokens).

    ext is None, or the dict of ptts_sampling_ext values (off: 0 / 0 / 1 / 0 / 0) when one of them changes the result.  The
    rules are the library's: `no_repeat_ngram_size` > 0 must be an int (<= 0 is off); `min_length` > 0 must be an int and is
    folded into min_new_tokens = max(0, min_length - n0), which a given `min_new_tokens` overrides (`_prepare_generated_length`);
    the warpers exist only with do_sample: `min_p` outside [0, 1] and `typical_p` <= 0 raise, `typical_p` >= 1 is off, and
    `epsilon_cutoff` / `eta_cutoff` outside (0, 1) are off without an error."""
    mnt = gc.min_new_tokens
    if mnt is None:
        ml = getattr(gc, "min_length", 0)
        if ml is not None and ml > 0:
            if not isinstance(ml, int):
                raise ValueError(f"`min_length` has to be a non-negative integer, but is {ml}")
            mnt = max(0, ml - int(n0))
    n = getattr(gc, "no_repeat_ngram_size", 0)
    if n is None or n <= 0:
        n = 0
    elif not isinstance(n, int):
        raise ValueError(f"`ngram_size` has to be a strictly positive integer, but is {n}")
    ext = dict(no_repeat_ngram_size=int(n), min_p=0.0, typical_p=1.0, epsilon_cutoff=0.0, eta_cutoff=0.0)
    if gc.do_sample:
        mp = getattr(gc, "min_p", None)
        if mp is not None:
            if not (0 <= mp <= 1.0):
                raise ValueError(f"`min_p` has to be a float in the [0, 1] interval, but is {mp}")
            ext["min_p"] = float(mp)
        tp = getattr(gc, "typical_p", 1.0)
        if tp is not None and tp < 1.0:
            if not float(tp) > 0:
                raise ValueError(f"`typical_p` has to be a float > 0 and < 1, but is {tp}")
            ext["typical_p"] = float(tp)
        for k in ("epsilon_cutoff", "eta_cutoff"):
            v = getattr(gc, k, 0.0)
            if v is not None and 0.0 < v < 1.0:
                ext[k] = float(v)
    active = ext["no_repeat_ngram_size"] > 0 or ext["min_p"] > 0 or ext["typical_p"] < 1 or ext["epsilon_cutoff"] > 0 or ext["eta_cutoff"] > 0
    return (ext if active else None), int(mnt or 0)


def no_repeat_ngram_mask(ids: torch.Tensor, scores: torch.Tensor, n: int) -> torch.Tensor:
    """NoRepeatNGramLogitsProcessor as torch ops: ids [R, cur_len] -> scores with the ids banned by repeated n-grams at -inf."""
    cur = ids.shape[1]
    if n <= 0 or cur < n:   # no complete n-gram yet
        return scores
    win = ids.unfold(1, n, 1)                                           # [R, cur - n + 1, n]
    match = (win[:, :, :n - 1] == ids[:, cur - n + 1:].unsqueeze(1)).all(-1)
    nxt = win[:, :, n - 1]
    ok = match & (nxt >= 0) & (nxt < scores.shape[1])
    hits = torch.zeros(scores.shape, dtype=torch.int32, device=scores.device)
    hits.scatter_add_(1, nxt.clamp(0, scores.shape[1] - 1), ok.to(torch.int32))
    return scores.masked_fill(hits > 0, -float("inf"))


def sampling_ext_warpers(scores: torch.Tensor, ext: dict) -> torch.Tensor:
    """transformers' MinP, Typical, Epsilon and Eta warpers as torch ops, in that order (min_tokens_to_keep = 1)."""
    ninf = -float("inf")
    if ext["min_p"] > 0:
        probs = scores.softmax(-1)
        rm = probs < ext["min_p"] * probs.amax(-1, keepdim=True)
        rm.scatter_(-1, probs.argmax(-1, keepdim=True), False)
        scores = scores.masked_fill(rm, ninf)
    if ext["typical_p"] < 1:
        nl = torch.log_softmax(scores, -1)
        ent = -(nl * nl.exp()).nansum(-1, keepdim=True)
        shifted = (-nl - ent).abs()
        ss, si = torch.sort(shifted, descending=False)
        cum = scores.gather(-1, si).softmax(-1).cumsum(-1)
        last = (cum < ext["typical_p"]).sum(1).clamp(max=ss.shape[-1] - 1)
        rm = ss > ss.gather(1, last.view(-1, 1))
        rm[..., :1] = False
        scores = scores.masked_fill(rm.scatter(1, si, rm), ninf)
    for k in ("epsilon_cutoff", "eta_cutoff"):
        eps = ext[k]
        if eps <= 0:
            continue
        probs = scores.softmax(-1)
        if k == "eta_cutoff":
            e = torch.tensor(eps, device=scores.device)
            ent = torch.distributions.Categorical(logits=scores).entropy()
            eps = torch.min(e, torch.sqrt(e) * torch.exp(-ent))[..., None]
        rm = (probs < eps) & (scores < scores.amax(-1, keepdim=True))
        scores = scores.masked_fill(rm, ninf)
    return scores


def _sequence_bias_dict(sb) -> dict:
    """SequenceBiasLogitsProcessor's argument checks (dict {tuple(ids): float} or list [[ids], float]) -> the dict it uses."""
    if not isinstance(sb, (dict, list)) or len(sb) == 0:
        raise ValueError(f"`sequence_bias` has to be a non-empty dictionary, or non-empty list of lists but is {sb}.")
    is_id = lambda t: isinstance(t, (int, np.integer)) and not isinstance(t, bool)
    if isinstance(sb, dict):
        if any(not isinstance(ids, tuple) for ids in sb):
            raise ValueError(f"`sequence_bias` has to be a dict with tuples as keys, but is {sb}.")
        if any(len(ids) == 0 or any(not is_id(t) or t < 0 for t in ids) for ids in sb):
            raise ValueError(f"Each key in `sequence_bias` has to be a non-empty tuple of positive integers, but is {sb}.")
        if any(not isinstance(b, float) for b in sb.values()):
            raise ValueError(f"`sequence_bias` has to be a dict with floats as values, but is {sb}.")
        return dict(sb)
    ok = lambda e: (isinstance(e, list) and len(e) == 2 and isinstance(e[0], list) and all(is_id(t) and t > 0 for t in e[0])
                    and isinstance(e[1], float))
    if any(not ok(e) for e in sb):
        raise ValueError(f"Each element in `sequence_bias` has to be a non-empty list of lists of positive integers and float, "
                         f"but is {sb}.")
    return {tuple(e[0]): e[1] for e in sb}


def _token_id(v, name: str, V: int) -> int:
    if isinstance(v, (list, tuple)) or (isinstance(v, torch.Tensor) and v.dim() > 0):
        if len(v) != 1:
            raise ValueError(f"`{name}` takes one id here, got {v}")
        v = v[0]
    if isinstance(v, torch.Tensor):
        if torch.is_floating_point(v):
            raise ValueError(f"`{name}` has to be a list of positive integers, but is {v}")
        v = int(v)
    if not isinstance(v, (int, np.integer)) or isinstance(v, bool) or v < 0:
        raise ValueError(f"`{name}` has to be a list of positive integers, but is {v}")
    if v >= V:
        raise ValueError(f"`{name}` {v} is outside the vocabulary of size {V}")
    return int(v)


def _id_list(v, name: str) -> list[int]:
    ids = list(v.tolist() if isinstance(v, torch.Tensor) else v)
    if any(not isinstance(t, (int, np.integer)) or isinstance(t, bool) for t in ids):
        raise ValueError(f"`{name}` has to be a list of integer ids, but is {v}")
    return [int(t) for t in ids]


class LogitsExt:
    """The ptts_logits_ext processors of one generate() call (resolve_logits_ext): their values, the device tables built from
    them once per call, and the same stages as torch ops for the host-driven loop.  In transformers' order: sequence_bias
    (before the n-gram bans and MinNewTokens), then forced BOS, forced EOS, InfNan, exponential decay, suppress, begin-suppress
    (before the Parler EOS processor), and LogitNormalization after the warpers."""

    def __init__(self, V: int, eos: int, max_length: int):
        self.V, self.eos, self.max_length = V, eos, max_length
        self.bias1 = None                   # np.float32 [V], or None
        self.seqs: list[tuple[tuple[int, ...], float]] = []   # the multi-id sequences in dict order (bias rounded to fp32)
        self.forced_bos = self.forced_eos = -1
        self.remove_invalid_values = self.renormalize_logits = False
        self.decay = None                   # np.float32 [max_length]: decay[c] = fp32(factor^(c - decay_start) - 1)
        self.decay_start = 0
        self.suppress = self.begin_suppress = None   # sorted in-vocabulary ids, or None
        self.begin_index = 1
        self._dev = None

    def active(self) -> bool:
        return (self.bias1 is not None or bool(self.seqs) or self.forced_bos >= 0 or self.forced_eos >= 0 or self.remove_invalid_values
                or self.decay is not None or self.suppress is not None or self.begin_suppress is not None or self.renormalize_logits)

    def c_struct(self, device) -> "_lib.LogitsExtC":
        """The C struct over device tables built once (they live as long as this object)."""
        if self._dev is None:
            W = (self.V + 31) // 32

            def bitmap(ids):
                if ids is None:
                    return None
                words = np.zeros(W, dtype=np.uint32)
                for t in ids:
                    words[t >> 5] |= np.uint32(1 << (t & 31))
                return torch.from_numpy(words.view(np.int32)).to(device)
            seq = np.zeros((max(1, len(self.seqs)), 1 + _lib.SEQ_BIAS_MAX_LEN), dtype=np.int32)
            for q, (ids, _) in enumerate(self.seqs):
                seq[q, 0] = len(ids)
                seq[q, 1:1 + len(ids)] = ids
            t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(device)
            self._dev = dict(bias1=t(self.bias1), seq=t(seq) if self.seqs else None,
                             seq_bias=t(np.array([b for _, b in self.seqs], dtype=np.float32)) if self.seqs else None,
                             decay=t(self.decay), suppress=bitmap(self.suppress), begin_suppress=bitmap(self.begin_suppress))
        d = self._dev
        return _lib.LogitsExtC(bias1=_lib.ptr(d["bias1"]), seq=_lib.ptr(d["seq"]), seq_bias=_lib.ptr(d["seq_bias"]),
                               n_seq=len(self.seqs), forced_bos_token_id=self.forced_bos, forced_eos_token_id=self.forced_eos,
                               remove_invalid_values=int(self.remove_invalid_values), decay=_lib.ptr(d["decay"]),
                               decay_start=self.decay_start, suppress=_lib.ptr(d["suppress"]),
                               begin_suppress=_lib.ptr(d["begin_suppress"]), begin_index=self.begin_index,
                               renormalize_logits=int(self.renormalize_logits))

    # -- the stages as torch ops (the host-driven loop); ids [R, cur_len] is the history, scores fp32 [R, V] --------------------
    def sequence_bias(self, ids: torch.Tensor, scores: torch.Tensor) -> torch.Tensor:
        if self.bias1 is None and not self.seqs:
            return scores
        bias = torch.zeros_like(scores)
        if self.bias1 is not None:
            bias += torch.from_numpy(self.bias1).to(scores.device)
        for seq, b in self.seqs:
            if len(seq) > ids.shape[1]:
                continue
            match = (ids[:, ids.shape[1] - len(seq) + 1:] == torch.tensor(seq[:-1], device=ids.device)).all(1)
            bias[:, seq[-1]] += torch.where(match, torch.tensor(b, device=scores.device), torch.tensor(0.0, device=scores.device))
        return scores + bias

    def before_parler(self, ids: torch.Tensor, scores: torch.Tensor) -> torch.Tensor:
        """forced BOS, forced EOS, InfNan, exponential decay, suppress, begin-suppress."""
        cur, ninf = ids.shape[1], -float("inf")
        for fid, col in ((self.forced_bos, 1), (self.forced_eos, self.max_length - 1)):
            if fid >= 0 and cur == col:
                scores = torch.full_like(scores, ninf)
                scores[:, fid] = 0
        if self.remove_invalid_values:
            fmax = torch.finfo(scores.dtype).max
            out = torch.where(scores != scores, 0.0, scores)
            out = torch.where(scores == float("inf"), fmax, out)
            scores = torch.where(scores == ninf, -fmax, out)
        if self.decay is not None and cur > self.decay_start:
            pen = torch.zeros_like(scores)
            pen[:, self.eos] = scores[:, self.eos].abs() * float(self.decay[cur])
            scores = scores + pen
        for ids_, on in ((self.suppress, True), (self.begin_suppress, cur == self.begin_index)):
            if ids_ is not None and on:
                scores = scores.masked_fill(torch.isin(torch.arange(scores.shape[1], device=scores.device),
                                                       torch.tensor(ids_, device=scores.device, dtype=torch.long)), ninf)
        return scores

    def normalize(self, scores: torch.Tensor) -> torch.Tensor:
        return scores.log_softmax(-1) if self.renormalize_logits else scores


def resolve_logits_ext(gc, n0: int, max_length: int, vocab_size: int, eos_token_id: int) -> Optional[LogitsExt]:
    """sequence_bias, suppress_tokens, begin_suppress_tokens, exponential_decay_length_penalty, forced_bos_token_id,
    forced_eos_token_id, remove_invalid_values and renormalize_logits from a GenerationConfig -> a LogitsExt, or None when none
    is set.  Greedy and sampling alike, as transformers builds them.  Raises ValueError where transformers raises (sequence_bias's
    format checks; a negative or float forced_eos_token_id), and up front for ids transformers only rejects when its processor
    first runs (sequence_bias or forced ids >= vocab_size).  Beyond transformers: more than PTTS_SEQ_BIAS_MAX multi-id sequences,
    one longer than PTTS_SEQ_BIAS_MAX_LEN, a forced_eos_token_id list of several ids, and a non-integer suppress id raise too.
    Suppress ids outside the vocabulary are ignored, as torch.isin ignores them."""
    V = int(vocab_size)
    lx = LogitsExt(V, int(eos_token_id), int(max_length))
    sb = getattr(gc, "sequence_bias", None)
    if sb is not None:
        sb = _sequence_bias_dict(sb)
        bad = [t for ids in sb for t in ids if t >= V]
        if bad:
            raise ValueError(f"The model vocabulary size is {V}, but the following tokens were being biased: {bad}")
        singles = {ids[0]: b for ids, b in sb.items() if len(ids) == 1}
        if singles:
            lx.bias1 = np.zeros(V, dtype=np.float32)
            for t, b in singles.items():
                lx.bias1[t] = np.float32(b)
        lx.seqs = [(tuple(int(t) for t in ids), float(np.float32(b))) for ids, b in sb.items() if len(ids) > 1]
        if len(lx.seqs) > _lib.SEQ_BIAS_MAX or any(len(s) > _lib.SEQ_BIAS_MAX_LEN for s, _ in lx.seqs):
            raise ValueError(f"`sequence_bias`: at most {_lib.SEQ_BIAS_MAX} sequences of 2 .. {_lib.SEQ_BIAS_MAX_LEN} ids are "
                             "supported by the device loop")
    fb = getattr(gc, "forced_bos_token_id", None)
    if fb is not None:
        lx.forced_bos = _token_id(fb, "forced_bos_token_id", V)
    fe = getattr(gc, "forced_eos_token_id", None)
    if fe is not None:
        lx.forced_eos = _token_id(fe, "forced_eos_token_id", V)
    lx.remove_invalid_values = getattr(gc, "remove_invalid_values", False) is True
    decay = getattr(gc, "exponential_decay_length_penalty", None)
    if decay is not None:
        if (not isinstance(decay, (tuple, list)) or len(decay) != 2 or not isinstance(decay[0], (int, np.integer))
                or not isinstance(decay[1], (int, float, np.number))):
            raise ValueError(f"`exponential_decay_length_penalty` has to be an (int start, float factor) pair, but is {decay}")
        lx.decay_start = int(decay[0]) + int(n0)   # regulation_start
        table = np.zeros(int(max_length), dtype=np.float32)
        with np.errstate(over="ignore"):
            for c in range(lx.decay_start + 1, int(max_length)):
                try:
                    table[c] = np.float32(pow(decay[1], c - lx.decay_start) - 1)   # Python's pow in double, rounded once
                except OverflowError:
                    table[c] = np.float32(np.inf)
        lx.decay = table
    for name in ("suppress_tokens", "begin_suppress_tokens"):
        v = getattr(gc, name, None)
        if v is not None:
            ids = sorted({t for t in _id_list(v, name) if 0 <= t < V})
            setattr(lx, "suppress" if name == "suppress_tokens" else "begin_suppress", ids if ids else None)
    # begin_index: the first generated column, one later when a forced BOS takes column 1 (_get_logits_processor)
    lx.begin_index = int(n0) + (1 if int(n0) == 1 and fb is not None else 0)
    lx.renormalize_logits = getattr(gc, "renormalize_logits", False) is True
    return lx if lx.active() else None


class ParlerTTSLogitsProcessor:
    """Stateful EOS gating across codebooks; HF LogitsProcessor protocol (__call__(input_ids, scores))."""

    def __init__(self, eos_token_id, num_codebooks: int, batch_size: int, device: str = "cuda"):
        if isinstance(eos_token_id, torch.Tensor):
            if torch.is_floating_point(eos_token_id) or (eos_token_id < 0).any():
                raise ValueError(f"`eos_token_id` has to be a list of positive integers, but is {eos_token_id}")
            eos_token_id = eos_token_id.reshape(-1).tolist()
        if isinstance(eos_token_id, int):
            eos_token_id = [eos_token_id]
        if len(eos_token_id) != 1 or eos_token_id[0] < 0:
            raise ValueError(f"`eos_token_id` has to be a list of positive integers, but is {eos_token_id}")
        self.eos_token_id = int(eos_token_id[0])
        self.batch_size, self.num_codebooks, self.device = batch_size, num_codebooks, device
        self.first_codebooks_unfinished = torch.arange(batch_size, device=device, dtype=torch.int64) * num_codebooks

    def __call__(self, input_ids: torch.LongTensor, scores: torch.FloatTensor) -> torch.FloatTensor:
        ids = input_ids.to(torch.int64).contiguous()
        if scores.dtype != torch.float32 or not scores.is_contiguous():
            raise ValueError("scores must be a contiguous float32 tensor (as `_sample` passes it)")
        _lib.check(_lib.lib().ptts_logits_processor(_lib.ptr(ids), ids.shape[0], ids.shape[1], ids.shape[1], _lib.ptr(scores),
                                                    scores.shape[1], self.eos_token_id, self.num_codebooks,
                                                    _lib.ptr(self.first_codebooks_unfinished), _lib.stream_ptr()))
        return scores  # mutated in place like the reference (:52)


# ---- decoder engine ------------------------------------------------------------------------------
def _decoder_config_c(cfg: ParlerTTSDecoderConfig, dtype: torch.dtype) -> _lib.DecoderConfigC:
    c = _lib.DecoderConfigC()
    c.hidden_size = cfg.hidden_size
    c.num_layers = cfg.num_hidden_layers
    c.num_heads = cfg.num_attention_heads
    c.num_kv_heads = cfg.num_key_value_heads
    c.num_cross_kv_heads = cfg.num_cross_attention_key_value_heads
    c.ffn_dim = cfg.ffn_dim
    c.vocab_size = cfg.vocab_size
    c.num_codebooks = cfg.num_codebooks
    c.max_positions = cfg.max_position_embeddings
    c.rope = 1 if cfg.rope_embeddings else 0
    if cfg.activation_function not in _ACT:
        raise ValueError(f"activation_function {cfg.activation_function!r} is not supported by the decoder kernels")
    c.activation = _ACT[cfg.activation_function]
    c.dtype = _lib.dtype_code(dtype)
    c.bos_token_id, c.pad_token_id, c.eos_token_id = cfg.bos_token_id, cfg.pad_token_id, cfg.eos_token_id
    c.rope_theta = float(cfg.rope_theta)
    c.layer_norm_eps = float(getattr(cfg, "layer_norm_eps", 1e-5))
    if cfg.hidden_size // cfg.num_attention_heads != 64:
        raise ValueError("the decoder kernels are specialised for head_dim == 64 (Parler-TTS Mini and Large)")
    return c


def _sinusoidal_table(n: int, dim: int) -> torch.Tensor:
    # ParlerTTSSinusoidalPositionalEmbedding.get_embedding semantics (:346-359): [cos | sin] halves
    half = dim // 2
    e = math.log(10000) / (half - 1)
    e = torch.exp(torch.arange(half, dtype=torch.int64).float() * -e)
    e = torch.arange(n, dtype=torch.int64).float().unsqueeze(1) * e.unsqueeze(0)
    return torch.cat([torch.cos(e), torch.sin(e)], dim=1)


def _rope_tables(cfg: ParlerTTSDecoderConfig):
    # ParlerTTSRotaryEmbedding (:380, :394-406): fp32 cos/sin of position x inv_freq, duplicated halves
    hd = cfg.hidden_size // cfg.num_attention_heads
    inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))
    fr = torch.arange(cfg.max_position_embeddings, dtype=torch.int64).float()[:, None] * inv[None, :]
    emb = torch.cat((fr, fr), dim=-1)
    return emb.cos(), emb.sin()


class DecoderEngine:
    """Packed decoder weights on one GPU + generation sessions.  One instance per model per device."""

    def __init__(self, cfg: ParlerTTSDecoderConfig, device, dtype: torch.dtype):
        self.cfg, self.device, self.dtype = cfg, torch.device(device), dtype
        self.c = _decoder_config_c(cfg, dtype)
        n = C.c_int64()
        _lib.check(_lib.lib().ptts_decoder_blob_bytes(C.byref(self.c), C.byref(n)))
        self.blob = torch.zeros(n.value, dtype=torch.uint8, device=self.device)
        self._sessions: dict[tuple, "GenSession"] = {}
        self._heads_rm: Optional[torch.Tensor] = None

    def heads_rowmajor(self) -> Optional[torch.Tensor]:
        """The folded lm heads row-major [K * V, H] for the fused scoring kernel (bf16; None for fp32, which scores unfused).
        A separate buffer (20 MB at Mini), made on the first scoring call."""
        if self.dtype != torch.bfloat16:
            return None
        if self._heads_rm is None:
            n = C.c_int64()
            _lib.check(_lib.lib().ptts_lm_heads_rowmajor_bytes(C.byref(self.c), C.byref(n)))
            buf = torch.empty(n.value, dtype=torch.uint8, device=self.device)
            _lib.check(_lib.lib().ptts_lm_heads_rowmajor_pack(C.byref(self.c), _lib.ptr(self.blob), _lib.ptr(buf), _lib.stream_ptr()))
            self._heads_rm = buf
        return self._heads_rm

    def _pack(self, tid: int, index: int, t: torch.Tensor):
        t = t.to(device=self.device)
        if t.dtype not in (torch.float32, torch.bfloat16):
            t = t.float()
        t = t.contiguous()
        rows, cols = (t.shape[0], t.numel() // t.shape[0]) if t.dim() >= 2 else (1, t.numel())
        _lib.check(_lib.lib().ptts_decoder_pack(C.byref(self.c), _lib.ptr(self.blob), tid, index, _lib.ptr(t),
                                                _lib.dtype_code(t.dtype), rows, cols, _lib.stream_ptr()))

    def load_state_dict(self, sd: dict[str, torch.Tensor], prefix: str = "decoder."):
        """sd uses the reference's parameter names (ParlerTTSForConditionalGeneration.state_dict())."""
        cfg, L = self.cfg, _lib
        p = prefix + "model.decoder."
        need = lambda k: sd[k] if k in sd else (_ for _ in ()).throw(ValueError(f"missing weight {k}"))
        for k in range(cfg.num_codebooks):
            self._pack(L.T_EMBED_TOKENS, k, need(f"{p}embed_tokens.{k}.weight"))
            self._pack(L.T_LM_HEAD, k, self._head(sd, prefix, k))
        if cfg.rope_embeddings:
            cos, sin = _rope_tables(cfg)
            self._pack(L.T_ROPE_COS, 0, cos)
            self._pack(L.T_ROPE_SIN, 0, sin)
        else:
            key = f"{p}embed_positions.weights"
            self._pack(L.T_POS_TABLE, 0, sd[key] if key in sd else _sinusoidal_table(cfg.max_position_embeddings, cfg.hidden_size))
        names = [("self_attn_layer_norm.weight", L.T_LN1_W), ("self_attn_layer_norm.bias", L.T_LN1_B),
                 ("self_attn.q_proj.weight", L.T_SELF_Q), ("self_attn.k_proj.weight", L.T_SELF_K),
                 ("self_attn.v_proj.weight", L.T_SELF_V), ("self_attn.out_proj.weight", L.T_SELF_O),
                 ("encoder_attn_layer_norm.weight", L.T_LN2_W), ("encoder_attn_layer_norm.bias", L.T_LN2_B),
                 ("encoder_attn.q_proj.weight", L.T_CROSS_Q), ("encoder_attn.k_proj.weight", L.T_CROSS_K),
                 ("encoder_attn.v_proj.weight", L.T_CROSS_V), ("encoder_attn.out_proj.weight", L.T_CROSS_O),
                 ("final_layer_norm.weight", L.T_LN3_W), ("final_layer_norm.bias", L.T_LN3_B),
                 ("fc1.weight", L.T_FC1), ("fc2.weight", L.T_FC2)]
        for i in range(cfg.num_hidden_layers):
            for nm, tid in names:
                self._pack(tid, i, need(f"{p}layers.{i}.{nm}"))
        self._pack(L.T_FINAL_LN_W, 0, need(p + "layer_norm.weight"))
        self._pack(L.T_FINAL_LN_B, 0, need(p + "layer_norm.bias"))
        _lib.check(_lib.lib().ptts_decoder_finalize(C.byref(self.c), _lib.ptr(self.blob), _lib.stream_ptr()))
        self._heads_rm = None   # repacked from the new weights at the next scoring call
        torch.cuda.current_stream().synchronize()
        return self

    def _head(self, sd, prefix, k):
        if f"{prefix}lm_heads.{k}.weight" in sd:
            return sd[f"{prefix}lm_heads.{k}.weight"]
        if f"{prefix}lm_heads.weight" in sd:  # use_fused_lm_heads (:1836): [K*V, H]
            V = self.cfg.vocab_size
            return sd[f"{prefix}lm_heads.weight"][k * V:(k + 1) * V]
        raise ValueError(f"missing weight {prefix}lm_heads.{k}.weight")

    def session(self, B: int, P: int, S: int, max_cache_len: int, max_input_len: int = 1, takes: int = 1) -> "GenSession":
        """max_input_len: the most decoder input columns (BOS column + code prefix) a generate() call on it may continue from.
        takes: consecutive rows that are takes of one description and share its cross-attention K/V (ptts_session_create3)."""
        key = (B, P, S)
        s = self._sessions.get(key)
        if s is None or s.max_cache_len < max_cache_len or s.max_input_len < max_input_len or s.takes != takes:
            if s is not None:
                s.close()
            s = GenSession(self, B, P, S, max_cache_len, max_input_len, takes)
            self._sessions = {key: s}  # keep one live session (the reference keeps one `_cache`, :3254-3309)
        return s


class GenSession:
    """Device-resident generation state for (B, P, S): KV caches, token history, processor state.  With takes > 1 the B rows are
    B / takes descriptions with `takes` consecutive takes each: prefill / score take B / takes encoder rows, everything else B."""

    def __init__(self, eng: DecoderEngine, B: int, P: int, S: int, max_cache_len: int, max_input_len: int = 1, takes: int = 1):
        self.eng, self.B, self.P, self.S, self.max_cache_len = eng, B, P, S, max_cache_len
        self.max_input_len, self.takes = int(max_input_len), int(takes)
        lib = _lib.lib()
        n = C.c_int64()
        _lib.check(lib.ptts_workspace_bytes3(C.byref(eng.c), B, P, S, max_cache_len, self.max_input_len, self.takes, C.byref(n)))
        self.ws = torch.zeros(n.value, dtype=torch.uint8, device=eng.device)
        h = C.c_void_p()
        _lib.check(lib.ptts_session_create3(C.byref(eng.c), _lib.ptr(eng.blob), _lib.ptr(self.ws), n.value, B, P, S,
                                            max_cache_len, self.max_input_len, self.takes, C.byref(h)))
        self.h = h
        self.K, self.V = eng.cfg.num_codebooks, eng.cfg.vocab_size
        self._keep: list[Any] = []
        self._forced = None
        self._outputs = None
        self._probes = None   # the buffers of the last ptts_generate_set_probes window (None: never set)
        self._input_ids = None
        self.n0 = 1

    def close(self):
        if self.h is not None:
            _lib.lib().ptts_session_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _view(self, fn, shape, dtype):
        p = C.c_void_p()
        _lib.check(fn(self.h, C.byref(p)))
        off = p.value - self.ws.data_ptr()
        n = int(torch.tensor(shape).prod()) * torch.empty((), dtype=dtype).element_size()
        return self.ws[off:off + n].view(dtype).view(*shape)

    @property
    def logits(self) -> torch.Tensor:
        return self._view(_lib.lib().ptts_session_logits, (self.B * self.K, self.V), torch.float32)

    @property
    def scores(self) -> torch.Tensor:
        return self._view(_lib.lib().ptts_session_scores, (self.B * self.K, self.V), torch.float32)

    @property
    def raw_ids(self) -> torch.Tensor:
        p, ld = C.c_void_p(), C.c_int32()
        _lib.check(_lib.lib().ptts_session_raw_ids(self.h, C.byref(p), C.byref(ld)))
        off = p.value - self.ws.data_ptr()
        return self.ws[off:off + self.B * self.K * ld.value * 8].view(torch.int64).view(self.B * self.K, ld.value)

    @property
    def state(self) -> torch.Tensor:
        """int32 [8]: cur_len, active, n_unfinished, done_blocks, steps_run, ..."""
        return self._view(_lib.lib().ptts_session_state, (8,), torch.int32)

    @property
    def eos_seen(self) -> torch.Tensor:
        """int32 [B * K]: 1 + the column of each row's first EOS, 0 while it has none."""
        return self._view(_lib.lib().ptts_session_eos_seen, (self.B * self.K,), torch.int32)

    @property
    def launches(self) -> int:
        n = C.c_int64()
        _lib.check(_lib.lib().ptts_session_launches(self.h, C.byref(n)))
        return n.value

    @property
    def fused(self) -> int:
        """0: decode steps use the multi-kernel path; 1: the fused persistent step kernel (one launch per token, step.cu);
        2: its cluster variant (step2.cu: one cluster per head, 6 device-wide phases per layer)."""
        n = C.c_int32()
        _lib.check(_lib.lib().ptts_session_fused(self.h, C.byref(n)))
        return n.value

    def begin(self, max_length: int, do_sample=False, temperature=1.0, top_k=0, top_p=1.0, min_new_tokens=0, seed=0,
              suppress_special=False, codebook_size=1024, row_base=0, input_ids: Optional[torch.Tensor] = None,
              ext: Optional[dict] = None, lext: Optional[LogitsExt] = None, input_lens: Optional[torch.Tensor] = None):
        """input_ids: None (the BOS column) or the BOS-led decoder input [B*K, n0] the generation continues from; the history
        then starts with its delayed form and the first sampled column is n0 (ptts_generate_begin_ids).
        input_lens: None, or [B] int32: row b continues from its first input_lens[b] columns (ptts_generate_begin_ids2); None
        when every row takes all n0.
        ext: None, or the ptts_sampling_ext values (resolve_sampling_ext) for this generation.
        lext: None, or the ptts_logits_ext processors (resolve_logits_ext); the session keeps it, and so its device tables, alive."""
        g = _lib.GenParamsC()
        g.max_length, g.min_new_tokens, g.do_sample = int(max_length), int(min_new_tokens or 0), int(bool(do_sample))
        g.top_k, g.top_p, g.temperature = int(top_k or 0), float(1.0 if top_p is None else top_p), float(temperature or 1.0)
        g.seed, g.suppress_special, g.codebook_size = int(seed) & (2 ** 64 - 1), int(bool(suppress_special)), int(codebook_size)
        g.row_base = int(row_base)  # global row of this shard's first (utterance, codebook) stream: Philox substream key
        if input_ids is None:
            self._input_ids, self.n0 = None, 1
            _lib.check(_lib.lib().ptts_generate_begin(self.h, C.byref(g), _lib.stream_ptr()))
        else:
            ids = input_ids.to(device=self.eng.device, dtype=torch.int64).contiguous()
            if ids.dim() != 2 or ids.shape[0] != self.B * self.K:
                raise ValueError(f"input_ids must be [{self.B * self.K}, n0], got {tuple(ids.shape)}")
            self._input_ids, self.n0 = ids, int(ids.shape[1])   # kept alive until the asynchronous begin kernel has read it
            if input_lens is None:
                _lib.check(_lib.lib().ptts_generate_begin_ids(self.h, C.byref(g), _lib.ptr(ids), self.n0, _lib.stream_ptr()))
            else:
                lens = input_lens.to(device=self.eng.device, dtype=torch.int32).contiguous()
                if tuple(lens.shape) != (self.B,):
                    raise ValueError(f"input_lens must be [{self.B}], got {tuple(lens.shape)}")
                _lib.check(_lib.lib().ptts_generate_begin_ids2(self.h, C.byref(g), _lib.ptr(ids), self.n0, _lib.ptr(lens),
                                                               _lib.stream_ptr()))
        if ext is not None:
            _lib.check(_lib.lib().ptts_generate_set_sampling_ext(self.h, C.byref(_lib.SamplingExtC(**ext))))
        self._lext = lext
        if lext is not None:
            _lib.check(_lib.lib().ptts_generate_set_logits_ext(self.h, C.byref(lext.c_struct(self.eng.device))))
        self._outputs = None   # the begin calls switch the per-step outputs off
        self.max_length = int(max_length)

    def prefill(self, prompt_hidden, prompt_mask, enc_hidden, enc_mask):
        dt, dev = self.eng.dtype, self.eng.device
        H = self.eng.cfg.hidden_size
        enc_hidden = enc_hidden.to(device=dev, dtype=dt).contiguous()
        if tuple(enc_hidden.shape) != (self.B // self.takes, self.S, H):
            raise ValueError(f"encoder states must be [{self.B // self.takes}, {self.S}, {H}], got {tuple(enc_hidden.shape)}")
        if self.P > 0:
            if prompt_hidden is None:
                raise ValueError("prompt_hidden_states are required for a session created with P > 0")
            prompt_hidden = prompt_hidden.to(device=dev, dtype=dt).contiguous()
            if tuple(prompt_hidden.shape) != (self.B, self.P, H):
                raise ValueError(f"prompt states must be [{self.B}, {self.P}, {H}], got {tuple(prompt_hidden.shape)}")
        pm = None if prompt_mask is None else prompt_mask.to(device=dev, dtype=torch.int64).contiguous()
        em = None if enc_mask is None else enc_mask.to(device=dev, dtype=torch.int64).contiguous()
        self._keep = [prompt_hidden, enc_hidden, pm, em]
        _lib.check(_lib.lib().ptts_prefill(self.h, _lib.ptr(prompt_hidden) if self.P > 0 else None, _lib.ptr(pm),
                                           _lib.ptr(enc_hidden), _lib.ptr(em), _lib.stream_ptr()))

    def score(self, prompt_hidden, prompt_mask, enc_hidden, enc_mask, dec_ids, labels, token_nll, logits=None, sums=None):
        """ptts_score: dec_ids [B * K, T] (as given), labels [B, T, K] or None -> token_nll [B, T, K], logits [B * K, T, V] and
        sums [K, 2] (per-codebook NLL sum and count) where given.  The session's caches are overwritten."""
        dt, dev = self.eng.dtype, self.eng.device
        H = self.eng.cfg.hidden_size
        enc_hidden = enc_hidden.to(device=dev, dtype=dt).contiguous()
        if tuple(enc_hidden.shape) != (self.B // self.takes, self.S, H):
            raise ValueError(f"encoder states must be [{self.B // self.takes}, {self.S}, {H}], got {tuple(enc_hidden.shape)}")
        if self.P > 0:
            prompt_hidden = prompt_hidden.to(device=dev, dtype=dt).contiguous()
            if tuple(prompt_hidden.shape) != (self.B, self.P, H):
                raise ValueError(f"prompt states must be [{self.B}, {self.P}, {H}], got {tuple(prompt_hidden.shape)}")
        pm = None if prompt_mask is None or self.P == 0 else prompt_mask.to(device=dev, dtype=torch.int64).contiguous()
        em = None if enc_mask is None else enc_mask.to(device=dev, dtype=torch.int64).contiguous()
        dec_ids = dec_ids.to(device=dev, dtype=torch.int64).contiguous()
        labels = None if labels is None else labels.to(device=dev, dtype=torch.int64).contiguous()
        heads = self.eng.heads_rowmajor() if (labels is not None and logits is None) else None
        self._keep = [prompt_hidden, enc_hidden, pm, em, dec_ids, labels]
        _lib.check(_lib.lib().ptts_score(self.h, _lib.ptr(prompt_hidden) if self.P > 0 else None, _lib.ptr(pm), _lib.ptr(enc_hidden),
                                         _lib.ptr(em), _lib.ptr(dec_ids), _lib.ptr(labels), int(dec_ids.shape[1]), _lib.ptr(heads),
                                         _lib.ptr(token_nll), _lib.ptr(logits), _lib.ptr(sums), _lib.stream_ptr()))

    def decode_forward(self):
        _lib.check(_lib.lib().ptts_decode_forward(self.h, _lib.stream_ptr()))

    def sample(self, forced: Optional[torch.Tensor] = None):
        f = None if forced is None else forced.to(device=self.eng.device, dtype=torch.int64).contiguous()
        self._forced = f   # keep the staging tensor alive until the next call (the launch is asynchronous); never accumulates
        _lib.check(_lib.lib().ptts_sample(self.h, _lib.ptr(f), _lib.stream_ptr()))

    def decode_steps(self, n: int):
        _lib.check(_lib.lib().ptts_decode_steps(self.h, int(n), _lib.stream_ptr()))

    def import_rows(self, src: "GenSession", src_rows: list[int], dst_rows: list[int]):
        """ptts_session_import_rows: row src_rows[i] of `src` (begun from the BOS column, prefilled, sampled) becomes slot
        dst_rows[i] of this session."""
        n = len(src_rows)
        if len(dst_rows) != n:
            raise ValueError(f"{n} source rows and {len(dst_rows)} destination rows")
        arr = lambda v: (C.c_int32 * max(n, 1))(*[int(x) for x in v])
        _lib.check(_lib.lib().ptts_session_import_rows(self.h, src.h, arr(src_rows), arr(dst_rows), n, _lib.stream_ptr()))

    def set_slots(self, cur_len: int, row_shift: list[int], row_key: list[int], row_max_length: Optional[list[int]] = None):
        """ptts_generate_set_slots2: slot mode, row b at its own column cur_len - row_shift[b] with Philox key row_key[b] and, when
        given, its own limit row_max_length[b] in [2K - 1, max_length] (None: every row max_length)."""
        if len(row_shift) != self.B or len(row_key) != self.B or (row_max_length is not None and len(row_max_length) != self.B):
            raise ValueError(f"row_shift, row_key and row_max_length must hold {self.B} entries")
        arr = lambda v: (C.c_int32 * self.B)(*[int(x) for x in v])
        lims = None if row_max_length is None else arr(row_max_length)
        _lib.check(_lib.lib().ptts_generate_set_slots2(self.h, int(cur_len), arr(row_shift), arr(row_key), lims, _lib.stream_ptr()))

    def set_outputs(self, logits: Optional[torch.Tensor], scores: Optional[torch.Tensor], first_step: int = 0, n_steps: int = 0,
                    step_stride: int = 0):
        """ptts_generate_set_outputs: the sampler records the raw logits and the processed scores of steps [first_step, first_step
        + n_steps) from the first element of `logits` / `scores` (fp32 CUDA tensors or views; None = not recorded), slot s of row r
        at (s - first_step) * step_stride + r * V floats.  Both None switches it off; generate_begin does too."""
        def addr(t):
            if t is None:
                return None
            if not t.is_cuda or t.dtype != torch.float32:
                raise ValueError("the output buffers must be float32 CUDA tensors")
            return C.c_void_p(t.data_ptr())
        self._outputs = (logits, scores)   # the buffers stay alive while the sampler may write them
        _lib.check(_lib.lib().ptts_generate_set_outputs(self.h, addr(logits), addr(scores), int(first_step), int(n_steps),
                                                        int(step_stride)))


    def set_probes(self, self_attn: Optional[torch.Tensor] = None, cross_attn: Optional[torch.Tensor] = None,
                   hidden: Optional[torch.Tensor] = None, first_step: int = 0, n_steps: int = 0, self_ld: int = 0):
        """ptts_generate_set_probes: the decoder passes write the attention weights and hidden states of steps [first_step,
        first_step + n_steps) (step 0: the prefill / score pass) into the given model-dtype CUDA tensors, each of which starts at
        this session's first batch row of slot first_step and steps by its stride(0) per slot.  All None switches it off."""
        def addr(t):
            if t is None:
                return None
            if not t.is_cuda or t.dtype != self.eng.dtype:
                raise ValueError(f"the probe buffers must be {self.eng.dtype} CUDA tensors")
            return C.c_void_p(t.data_ptr())
        step = lambda t: 0 if t is None or t.dim() == 0 else int(t.stride(0))
        bufs = (self_attn, cross_attn, hidden)
        self._probes = None if all(t is None for t in bufs) else bufs   # the buffers stay alive while the kernels may write them
        _lib.check(_lib.lib().ptts_generate_set_probes(self.h, addr(self_attn), addr(cross_attn), addr(hidden), int(first_step),
                                                       int(n_steps), int(self_ld), step(self_attn), step(cross_attn), step(hidden)))

    def set_alignment(self, heads: Optional[torch.Tensor] = None, key0: int = 0, key_len: int = 0, out: Optional[torch.Tensor] = None,
                      first_row: int = 0, n_rows: int = 0):
        """ptts_generate_set_alignment: decode steps write the alignment rows [first_row, first_row + n_rows) of the [n_heads, 2]
        int32 (layer, head) list over keys [key0, key0 + key_len) into out [n_rows, B, key_len] fp32.  out None switches it off."""
        if out is None:
            self._align = None
            _lib.check(_lib.lib().ptts_generate_set_alignment(self.h, None, 0, 0, 0, None, 0, 0))
            return
        if out.dtype != torch.float32 or tuple(out.shape) != (n_rows, self.B, key_len):
            raise ValueError(f"the alignment buffer must be float32 [{n_rows}, {self.B}, {key_len}]")
        self._align = (heads, out)   # the list and the buffer stay alive while the kernels may read / write them
        _lib.check(_lib.lib().ptts_generate_set_alignment(self.h, _lib.ptr(heads), int(heads.shape[0]), int(key0), int(key_len),
                                                          _lib.ptr(out), int(first_row), int(n_rows)))


def output_window(step: int, chunk: int) -> tuple[int, int]:
    """The chunk of generate()'s per-step outputs that holds `step`: (index, first step)."""
    return step // chunk, (step // chunk) * chunk


def steps_in_window(step: int, steps_left: int, chunk: int) -> int:
    """Decode steps to enqueue from `step` on: up to steps_left, without crossing a chunk boundary, so one ptts_decode_steps call
    writes inside one output window."""
    return min(chunk - step % chunk, steps_left)


class StepOutputs:
    """generate()'s `scores` / `logits`: one fp32 [rows, V] block per generated column, kept in chunks of CHUNK steps (the device
    loop's chunk).  A chunk is allocated NaN-filled when a loop first reaches it, so nothing is sized by max_length up front.  The
    shards of one batch share the chunks and write their own rows; a shard that ended leaves its rows NaN."""
    CHUNK = 64

    def __init__(self, rows: int, vocab_size: int, device, scores: bool, logits: bool):
        self.rows, self.V, self.device = int(rows), int(vocab_size), device
        self.chunks = {k: [] for k, on in (("scores", scores), ("logits", logits)) if on}

    def chunk(self, c: int) -> dict:
        for lst in self.chunks.values():
            while len(lst) <= c:
                lst.append(torch.full((self.CHUNK, self.rows, self.V), float("nan"), dtype=torch.float32, device=self.device))
        return {k: lst[c] for k, lst in self.chunks.items()}

    def attach_prefill(self, sess: "GenSession", b0: int):
        pass   # the prefill records no row: step 0 is the sample after it

    def attach_window(self, sess: "GenSession", step: int, b0: int):
        """Points the session's sampler at the chunk holding `step`, at the rows of batch row b0 on."""
        c, first = output_window(step, self.CHUNK)
        ch = self.chunk(c)
        at = lambda k: ch[k][0, b0 * sess.K] if k in ch else None
        sess.set_outputs(at("logits"), at("scores"), first, self.CHUNK, self.rows * self.V)

    def detach(self, sess: "GenSession", b0: int):
        sess.set_outputs(None, None)   # the session keeps no reference to the chunks

    def put(self, step: int, row0: int, logits: torch.Tensor, scores: torch.Tensor):
        """Stores one step's rows from torch (the host-driven loop)."""
        c, first = output_window(step, self.CHUNK)
        ch = self.chunk(c)
        for k, t in (("logits", logits), ("scores", scores)):
            if k in ch:
                ch[k][step - first, row0:row0 + t.shape[0]].copy_(t)

    def result(self, n_steps: int) -> dict:
        """{"scores": tuple of n_steps [rows, V] views, "logits": ...} for the outputs asked for."""
        C_ = self.CHUNK
        if n_steps > 0:
            self.chunk((n_steps - 1) // C_)
        return {k: tuple(lst[t // C_][t % C_] for t in range(n_steps)) for k, lst in self.chunks.items()}


class StepProbes:
    """generate()'s output_attentions / output_hidden_states, written by the decoder passes in the model dtype.

    Entry 0 (the prefill, q = P + n0 rows) has buffers of its own; the decode steps t >= 1 (q = 1) live in the chunks of
    StepOutputs.CHUNK steps that the device loop already cuts its calls at.  Chunk c holds, per step, self-attention rows
    [B, L, heads, T_hi(c)] with T_hi(c) = P + n0 + the chunk's last step (the longest row in it), cross-attention rows
    [B, L, heads, S] and hidden rows [B, L + 1, H]; it is allocated NaN-filled when a loop first reaches it, and the entries are
    views narrowed to their own T_kv = P + n0 + t.  Batch rows are outermost, so shards write their own rows; a shard that ended
    leaves its rows NaN.  Memory is what the entries hold: the self-attention alone is L * B * heads * sum(T_kv) * 2 bytes in
    bf16 (10 s of Parler-TTS-Mini audio, ~860 steps: ~0.3 GB per utterance, ~10 GB at B = 32), the order of the reference's."""
    CHUNK = StepOutputs.CHUNK

    def __init__(self, n_layers: int, batch: int, heads: int, S: int, H: int, P: int, n0: int, dtype, device, attentions: bool,
                 hidden: bool, chunk: int = CHUNK):
        """chunk: steps per chunk (generate(): StepOutputs.CHUNK; 1 for one step of the step operator, which then holds that
        step's rows only, each exactly its T_kv long)."""
        self.CHUNK = int(chunk)
        self.L, self.B, self.nh, self.S, self.H, self.P, self.n0 = n_layers, batch, heads, S, H, P, n0
        self.dtype, self.device, self.attn, self.hid = dtype, device, bool(attentions), bool(hidden)
        self.entry0 = None
        self.chunks: dict[int, dict] = {}

    def _full(self, *shape):
        return torch.full(shape, float("nan"), dtype=self.dtype, device=self.device)

    def t_hi(self, c: int) -> int:
        return self.P + self.n0 + (c + 1) * self.CHUNK - 1

    def _entry0(self) -> dict:
        if self.entry0 is None:
            q, L, B = self.P + self.n0, self.L, self.B
            self.entry0 = {}
            if self.attn:
                self.entry0["self"] = self._full(1, B, L, self.nh, q, q)
                self.entry0["cross"] = self._full(1, B, L, self.nh, q, self.S)
            if self.hid:
                self.entry0["hidden"] = self._full(1, B, L + 1, q, self.H)
        return self.entry0

    def chunk(self, c: int) -> dict:
        if c not in self.chunks:
            L, B, n = self.L, self.B, self.CHUNK
            ch = {}
            if self.attn:
                ch["self"] = self._full(n, B, L, self.nh, self.t_hi(c))
                ch["cross"] = self._full(n, B, L, self.nh, self.S)
            if self.hid:
                ch["hidden"] = self._full(n, B, L + 1, self.H)
            self.chunks[c] = ch
        return self.chunks[c]

    def attach_prefill(self, sess: "GenSession", b0: int):
        """Points the session's prefill at entry 0, from batch row b0 on."""
        e = self._entry0()
        at = lambda k: e[k][:, b0] if k in e else None
        sess.set_probes(at("self"), at("cross"), at("hidden"), 0, 1, self.P + self.n0)

    def attach_window(self, sess: "GenSession", step: int, b0: int):
        """Points the session's decode steps at the chunk holding `step`, from batch row b0 on (step 0 is entry 0: nothing)."""
        if step == 0:
            return
        c, first = output_window(step, self.CHUNK)
        f = max(first, 1)   # (slot 0 of chunk 0 stays unused: step 0 is entry 0)
        ch = self.chunk(c)
        at = lambda k: ch[k][f - first:, b0] if k in ch else None
        sess.set_probes(at("self"), at("cross"), at("hidden"), f, first + self.CHUNK - f, self.t_hi(c))

    def detach(self, sess: "GenSession", b0: int):
        sess.set_probes()   # the session keeps no window (nor the chunks) past the call

    def entry(self, t: int) -> dict:
        """Entry t: decoder_attentions / cross_attentions (tuples of L [B, heads, q, T_kv] / [B, heads, q, S]) and
        decoder_hidden_states (a tuple of L + 1 [B, q, H]), for the outputs asked for (views; NaN where nothing was written)."""
        L, out = self.L, {}
        if t == 0:
            e = self._entry0()
            sa, ca, hs = (e.get(k) for k in ("self", "cross", "hidden"))
            if self.attn:
                out["decoder_attentions"] = tuple(sa[0, :, l] for l in range(L))
                out["cross_attentions"] = tuple(ca[0, :, l] for l in range(L))
            if self.hid:
                out["decoder_hidden_states"] = tuple(hs[0, :, i] for i in range(L + 1))
            return out
        ch, i = self.chunk(t // self.CHUNK), t % self.CHUNK
        if self.attn:
            out["decoder_attentions"] = tuple(ch["self"][i, :, l, :, None, :self.P + self.n0 + t] for l in range(L))
            out["cross_attentions"] = tuple(ch["cross"][i, :, l, :, None, :] for l in range(L))
        if self.hid:
            out["decoder_hidden_states"] = tuple(ch["hidden"][i, :, j, None, :] for j in range(L + 1))
        return out

    def result(self, n_steps: int) -> dict:
        """The entries 0 .. n_steps - 1 as transformers' tuples (one entry per generated column)."""
        entries = [self.entry(t) for t in range(n_steps)]
        return {k: tuple(e[k] for e in entries) for k in (entries[0] if entries else {})}


# ---- model classes -------------------------------------------------------------------------------
def resolve_alignment_heads(heads, n_layers: int, n_heads: int) -> list[list[int]]:
    """GenerationConfig.alignment_heads -> the [layer, head] pairs return_token_timestamps averages.  None: every head of the last
    ceil(n_layers / 2) layers (openai-whisper's choice when a model has no known alignment heads; no Parler checkpoint has any).
    An empty list, a pair outside the decoder or a pair listed twice raises ValueError."""
    if heads is None:
        return [[l, h] for l in range(n_layers // 2, n_layers) for h in range(n_heads)]
    try:
        pairs = [list(p) for p in heads]
    except TypeError:
        raise ValueError(f"`alignment_heads` must be a list of [layer, head] pairs, got {heads!r}") from None
    if not pairs:
        raise ValueError("`alignment_heads` is empty: list at least one [layer, head] pair, or None for the default heads")
    seen = set()
    for p in pairs:
        if len(p) != 2 or not all(isinstance(v, int) and not isinstance(v, bool) for v in p):
            raise ValueError(f"`alignment_heads` must be a list of [layer, head] integer pairs, got {p!r}")
        l, h = p
        if not (0 <= l < n_layers and 0 <= h < n_heads):
            raise ValueError(f"`alignment_heads` pair {p} is outside the decoder's {n_layers} layers x {n_heads} heads")
        if (l, h) in seen:
            raise ValueError(f"`alignment_heads` lists {p} twice")
        seen.add((l, h))
    return pairs


def token_frames(raw_ids: torch.Tensor, n0: int, num_codebooks: int, codebook_size: int) -> torch.Tensor:
    """raw_ids [B * K, T] -> int32 [B]: the generated frames of each utterance that token timestamps align to.  Generated frame f
    is codebook 0's id at column n0 + f and codebook k's at column n0 + f + k (the delay pattern); the frames counted are the
    leading ones whose K ids are all codes (< codebook_size, as the audio decode requires), so they end at the utterance's EOS,
    at the last frame every codebook reaches (T - n0 - K + 1) and at the last column that got an alignment row (T - n0 - 1)."""
    K = num_codebooks
    T = raw_ids.shape[1] - n0
    F = max(0, min(T - K + 1, T - 1))
    r = raw_ids.view(-1, K, raw_ids.shape[1])
    ok = torch.ones(r.shape[0], F, dtype=torch.bool, device=raw_ids.device)
    for k in range(K):
        ok &= r[:, k, n0 + k:n0 + k + F] < codebook_size
    return ok.int().cumprod(dim=1).sum(dim=1).to(torch.int32)


def align_dtw(alignment: torch.Tensor, n_frames: torch.Tensor, key_mask: Optional[torch.Tensor] = None):
    """ptts_align_dtw: alignment [B, T, P] fp32 (CUDA) -> (filtered [B, T, P]: the width-7 median along each utterance's first
    n_frames[b] frames, NaN past them; jumps [B, P] int32: the first frame of each unmasked key on the DTW path of -filtered,
    -1 for a masked key).  openai-whisper's median filter and DTW as transformers' generation_whisper runs them."""
    B, T, P = alignment.shape
    dev = alignment.device
    x = alignment.to(torch.float32).contiguous()
    nf = n_frames.to(device=dev, dtype=torch.int32).contiguous()
    km = None if key_mask is None else key_mask.to(device=dev, dtype=torch.int32).contiguous()
    filtered = torch.full_like(x, float("nan"))
    trace = torch.empty(B * (P + 1) * (T + 1), dtype=torch.uint8, device=dev)
    jumps = torch.empty(B, P, dtype=torch.int32, device=dev)
    _lib.check(_lib.lib().ptts_align_dtw(_lib.ptr(x), B, T, P, _lib.ptr(nf), _lib.ptr(km), _lib.ptr(filtered), _lib.ptr(trace),
                                         _lib.ptr(jumps), _lib.stream_ptr()))
    return filtered, jumps


class StepAlignment:
    """generate()'s return_token_timestamps recorder: row t of utterance b (alignment[b, t]) is the alignment heads' mean
    distribution over the key_len transcript keys for the query of generated column n0 + t, written by the decode step whose
    input is that column (ptts_generate_set_alignment).  The last generated column is never a decode step's input, so its row,
    and the rows of a shard that ended before the longest one, stay NaN.  One [rows, B_shard, key_len] buffer and window per session."""
    CHUNK = None   # the window spans the whole call

    def __init__(self, heads: list[list[int]], batch: int, rows: int, key0: int, key_len: int, device):
        self.heads = torch.tensor(heads, dtype=torch.int32, device=device).reshape(-1, 2).contiguous()
        self.rows, self.key0, self.key_len = rows, key0, key_len
        self.alignment = torch.full((batch, rows, key_len), float("nan"), dtype=torch.float32, device=device)

    def attach_prefill(self, sess: "GenSession", b0: int):
        self.buf = torch.full((self.rows, sess.B, self.key_len), float("nan"), dtype=torch.float32, device=self.alignment.device)
        sess.set_alignment(self.heads, self.key0, self.key_len, self.buf, 0, self.rows)

    def attach_window(self, sess: "GenSession", step: int, b0: int):
        pass

    def detach(self, sess: "GenSession", b0: int):
        sess.set_alignment()
        self.alignment[b0:b0 + self.buf.shape[1]] = self.buf.permute(1, 0, 2)
        self.buf = None


@contextlib.contextmanager
def recording(sess: "GenSession", recorders, b0: int, step: int = 0):
    """Attaches the recorders (StepOutputs, StepProbes, StepAlignment; rows from batch row b0 on) for the prefill / score pass
    (step 0) or for the decode step `step`, and detaches them and collects their rows when the block ends, whatever happens in it
    (in reverse order).  A token loop in the block moves their windows: attach_window(sess, t, b0) before the steps from t on."""
    attached = []
    try:
        for r in recorders:
            if step == 0:
                r.attach_prefill(sess, b0)
            else:
                r.attach_window(sess, step, b0)
            attached.append(r)
        yield
    finally:
        for r in reversed(attached):
            r.detach(sess, b0)


class Sampling(NamedTuple):
    """One generate() call's sampling settings (ParlerTTSForConditionalGeneration._sampling): what GenSession.begin takes (a
    shard begins at row_base + its first row * K), and the caller's logits processors and stopping criteria (the host-driven
    loop runs the call when there are any)."""
    max_length: int
    do_sample: bool
    temperature: float
    top_k: int
    top_p: float
    min_new_tokens: int
    seed: int
    suppress_special: bool
    codebook_size: int
    row_base: int
    ext: Optional[dict]           # resolve_sampling_ext
    lext: Optional[LogitsExt]     # resolve_logits_ext
    processors: list
    criteria: list


class GenerateOutput(dict):
    """Stands in for HF's GenerateEncoderDecoderOutput: .sequences plus ["audios_length"] (:3648-3651)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


class ParlerTTSSeq2SeqLMOutput(GenerateOutput):
    """ParlerTTSForConditionalGeneration.forward's result: loss, per_codebook_losses (K scalars), token_losses [B, T, K] (the NLL
    of each counted label, 0 elsewhere), logits [B * K, T, V] (None when labels are given without return_logits=True) and
    encoder_last_hidden_state."""


class ParlerTTSCache:
    """`past_key_values` of ParlerTTSForCausalLM.forward: the device session that owns the pre-allocated self-attention K/V
    cache (append in place at cache_position) and the cross-attention K/V projected once at the first call -- the roles of
    EncoderDecoderCache(StaticCache, StaticCache) in the reference (:3254-3309)."""

    def __init__(self, session: "GenSession"):
        self.session = session
        self.steps = 0

    def get_seq_length(self) -> int:
        return self.session.P + 1 + self.steps

    def get_max_cache_shape(self) -> int:
        return self.session.max_cache_len


class ParlerTTSForCausalLM:
    """Decoder + K LM heads as a step operator over a KV-cached session (reference :1824-1974)."""

    def __init__(self, config: ParlerTTSDecoderConfig, device="cuda", dtype=torch.bfloat16):
        self.config = config
        self.num_codebooks = config.num_codebooks
        self.vocab_size = config.vocab_size
        self.device, self.dtype = torch.device(device), dtype
        self.engine = DecoderEngine(config, device, dtype)

    def load_state_dict(self, sd, prefix=""):
        self.engine.load_state_dict(sd, prefix=prefix)
        return self

    def build_delay_pattern_mask(self, input_ids, bos_token_id, pad_token_id, max_length):
        return build_delay_pattern_mask(input_ids, bos_token_id, pad_token_id, max_length, self.num_codebooks)

    @torch.no_grad()
    def forward(self, input_ids: torch.LongTensor = None, attention_mask=None, encoder_hidden_states=None,
                encoder_attention_mask=None, prompt_hidden_states=None, prompt_attention_mask=None, past_key_values=None,
                use_cache: bool = True, cache_position=None, return_dict: bool = True, max_cache_len: Optional[int] = None,
                output_attentions: bool = False, output_hidden_states: bool = False, **kwargs):
        """The step operator an HF-style loop calls (reference :1865-1974): input_ids [B*K, 1] (delay mask already applied, as
        prepare_inputs_for_generation does at :2909) -> logits [B*K, 1, V], over a KV cache kept in `past_key_values`.

        * first call (past_key_values None): `encoder_hidden_states` [B, S, H] (already multiplied by their mask) and optionally
          `prompt_hidden_states` [B, P, H] are required; the prompt prefix + the given ids go through ptts_prefill and a
          ParlerTTSCache (the session: pre-allocated self- and cross-attention K/V) is returned as `past_key_values`.
          Only the LAST position's logits are materialised (what `_sample` reads): shape [B*K, 1, V], not [B*K, P+1, V].
        * later calls: the ids are appended (ptts_sample with forced tokens) and one cached step runs on the fused kernel
          (ptts_decode_forward).
        Inputs longer than one column, `inputs_embeds`, `labels` and `use_cache=False` belong to training / the no-cache path and
        are outside this operator (ValueError).
        output_attentions / output_hidden_states add this call's `attentions` / `cross_attentions` (L x [B, heads, q, T_kv] /
        [B, heads, q, S]) and `hidden_states` (L+1 x [B, q, H]), q = P + 1 at the first call and 1 after it (the weights by the
        reference's eager definition, see ParlerTTSForConditionalGeneration.generate); the step then runs the multi-kernel
        path, with the same logits."""
        if kwargs.get("inputs_embeds") is not None or kwargs.get("labels") is not None or not use_cache:
            raise ValueError("ParlerTTSForCausalLM.forward on this path is the cached decode-step operator: input_ids [B*K, 1], use_cache=True")
        if input_ids is None or input_ids.dim() != 2 or input_ids.shape[1] != 1 or input_ids.shape[0] % self.num_codebooks != 0:
            raise ValueError(f"input_ids must be [batch * num_codebooks, 1], got {None if input_ids is None else tuple(input_ids.shape)}")
        B = input_ids.shape[0] // self.num_codebooks
        ids = input_ids[:, 0].to(self.device, torch.int64).contiguous()
        if past_key_values is None:
            if encoder_hidden_states is None:
                raise ValueError("the first call needs `encoder_hidden_states`")
            S = encoder_hidden_states.shape[1]
            P = 0 if prompt_hidden_states is None else prompt_hidden_states.shape[1]
            cap = int(max_cache_len or self.config.max_position_embeddings)
            sess = GenSession(self.engine, B, P, S, cap)   # an independent cache, not the engine's shared generate() session
            sess.begin(cap - P, do_sample=False)
            if not bool((ids == self.config.bos_token_id).all()):
                raise ValueError("the first call must feed the decoder start (BOS) column")
            probes = self._probes(B, P, S, output_attentions, output_hidden_states)
            with recording(sess, [] if probes is None else [probes], 0):
                sess.prefill(prompt_hidden_states, prompt_attention_mask if P > 0 else None, encoder_hidden_states, encoder_attention_mask)
            past_key_values = ParlerTTSCache(sess)
        else:
            if not isinstance(past_key_values, ParlerTTSCache) or past_key_values.session.B != B:
                raise ValueError("past_key_values must be the ParlerTTSCache returned by the first call (same batch)")
            sess = past_key_values.session
            sess.sample(forced=ids)
            step = past_key_values.steps + 1
            probes = self._probes(B, sess.P, sess.S, output_attentions, output_hidden_states)
            with recording(sess, [] if probes is None else [probes], 0, step):
                sess.decode_forward()
            past_key_values.steps += 1
        logits = sess.logits.clone().unsqueeze(1)   # [B*K, 1, V] fp32
        if not return_dict:
            return (logits, past_key_values)
        out = GenerateOutput(logits=logits, past_key_values=past_key_values)
        if probes is not None:
            names = dict(decoder_attentions="attentions", cross_attentions="cross_attentions", decoder_hidden_states="hidden_states")
            out.update({names[k]: v for k, v in probes.entry(past_key_values.steps).items()})
        return out

    def _probes(self, B, P, S, attentions, hidden):
        """A StepProbes for one call of the step operator, or None when nothing is asked: chunks of one step, so a decode
        step's entry is exactly its own rows (its self-attention T_kv long) and keeps nothing else alive."""
        if not (attentions or hidden):
            return None
        c = self.config
        return StepProbes(c.num_hidden_layers, B, c.num_attention_heads, S, c.hidden_size, P, 1, self.dtype, self.device,
                          attentions, hidden, chunk=1)

    __call__ = forward

    @staticmethod
    def apply_delay_pattern_mask(input_ids, decoder_pad_token_mask):
        return apply_delay_pattern_mask(input_ids, decoder_pad_token_mask)


class ParlerTTSForConditionalGeneration:
    """generate(): description/prompt conditioning -> audio tokens -> waveform, hot path on sm_90a kernels."""

    config_class = ParlerTTSConfig
    main_input_name = "input_ids"
    # model kwargs generate() understands (reference: _validate_model_kwargs over forward()'s signature)
    _MODEL_KWARGS = frozenset({"input_ids", "attention_mask", "prompt_input_ids", "prompt_attention_mask", "prompt_hidden_states",
                               "encoder_outputs", "input_values", "decoder_input_ids", "decoder_attention_mask", "padding_mask",
                               "use_cache", "cache_implementation", "output_attentions", "output_hidden_states"})
    # GenerationConfig fields the device loop does not implement, with the value that means "off"
    _NEUTRAL_GENERATION_KNOBS = {"num_beam_groups": 1, "repetition_penalty": 1.0, "length_penalty": 1.0,
                                 "penalty_alpha": None, "bad_words_ids": None, "force_words_ids": None, "guidance_scale": None}

    def __init__(self, config: ParlerTTSConfig, device="cuda", dtype=torch.bfloat16, text_encoder=None):
        if not isinstance(config, ParlerTTSConfig):
            raise ValueError(f"Config: {config} has to be of type {self.config_class}")
        self.config = config
        self.device, self.dtype = torch.device(device), dtype
        self.decoder = ParlerTTSForCausalLM(config.decoder, device, dtype)
        self.audio_encoder = DACModel(config.audio_encoder, device, dtype)
        self.text_encoder = text_encoder  # a torch module (T5 encoder) or None; not part of the replaced path
        self.prompt_cross_attention = bool(config.prompt_cross_attention)
        # Side-input parameters exist (zero-filled) from construction on, with shapes that depend on the config only, so every
        # rank of a sharded run issues the SAME list of broadcasts at init (dist.broadcast_model_weights); `_side_loaded`
        # says whether they hold real weights.  enc_to_dec_proj exists iff the text encoder's width differs (:2388-2392).
        dd = config.decoder
        self.embed_prompts_weight: torch.Tensor = torch.zeros(config.vocab_size, dd.hidden_size, device=self.device, dtype=dtype)
        # prompt_cross_attention: the prompt's sinusoidal positions (embed_positions.weights, :2397-2402), valid from construction
        # on; a checkpoint's own table replaces it at load_state_dict
        self.embed_positions_weight: Optional[torch.Tensor] = None
        if self.prompt_cross_attention:
            self.embed_positions_weight = _sinusoidal_table(dd.max_position_embeddings, dd.hidden_size).to(self.device, dtype)
        te_hidden = (config.text_encoder or {}).get("d_model", (config.text_encoder or {}).get("hidden_size"))
        self.enc_to_dec_proj: Optional[tuple] = None
        if te_hidden is not None and int(te_hidden) != dd.hidden_size:
            self.enc_to_dec_proj = (torch.zeros(dd.hidden_size, int(te_hidden), device=self.device, dtype=dtype),
                                    torch.zeros(dd.hidden_size, device=self.device, dtype=dtype))
        self._side_loaded = False
        self.use_audio_scales = True   # DACModel.decode has an `audio_scales` parameter (:2416-2417)
        self.use_4dim_audio_codes = True  # dac_on_the_hub (:2419-2422, quirk Q14)
        d = config.decoder
        self.generation_config = GenerationConfig(
            max_length=int(30 * config.audio_encoder.frame_rate), do_sample=True, bos_token_id=d.bos_token_id,
            pad_token_id=d.pad_token_id, eos_token_id=d.eos_token_id, decoder_start_token_id=d.bos_token_id)

    # -- weights -----------------------------------------------------------------------------------
    def load_state_dict(self, sd: dict[str, torch.Tensor], dac_state_dict: Optional[dict] = None):
        self.decoder.engine.load_state_dict(sd, prefix="decoder.")
        if "embed_prompts.weight" in sd:
            w = sd["embed_prompts.weight"].to(self.device, self.dtype)
            if w.shape == self.embed_prompts_weight.shape:
                self.embed_prompts_weight.copy_(w)
            else:  # a checkpoint whose text vocabulary differs from config.vocab_size: follow the checkpoint
                self.embed_prompts_weight = w.contiguous()
            self._side_loaded = True
        if "enc_to_dec_proj.weight" in sd:
            w, b = sd["enc_to_dec_proj.weight"].to(self.device, self.dtype), sd["enc_to_dec_proj.bias"].to(self.device, self.dtype)
            if self.enc_to_dec_proj is not None and self.enc_to_dec_proj[0].shape == w.shape:
                self.enc_to_dec_proj[0].copy_(w); self.enc_to_dec_proj[1].copy_(b)
            else:
                self.enc_to_dec_proj = (w.contiguous(), b.contiguous())
        if self.embed_positions_weight is not None and "embed_positions.weights" in sd:
            w = sd["embed_positions.weights"]
            if tuple(w.shape) != tuple(self.embed_positions_weight.shape):
                raise ValueError(f"embed_positions.weights must be {tuple(self.embed_positions_weight.shape)} "
                                 f"(max_position_embeddings x hidden_size), got {tuple(w.shape)}")
            self.embed_positions_weight.copy_(w.to(self.device, self.dtype))
        ae = {k[len("audio_encoder."):]: v for k, v in sd.items() if k.startswith("audio_encoder.")}
        if dac_state_dict is not None:
            ae = dac_state_dict
        if ae:
            self.audio_encoder.load_state_dict(ae)
        return self

    @classmethod
    def from_pretrained(cls, path: str, device="cuda", torch_dtype=torch.bfloat16, **kwargs):
        """Load a local reference checkpoint directory (config.json + *.safetensors)."""
        config = ParlerTTSConfig.from_pretrained(path)
        from safetensors.torch import load_file
        sd = {}
        for f in sorted(os.listdir(path)):
            if f.endswith(".safetensors"):
                sd.update(load_file(os.path.join(path, f)))
        if not sd:
            raise ValueError(f"no .safetensors weights found under {path}")
        text_encoder = None
        te = {k[len("text_encoder."):]: v for k, v in sd.items() if k.startswith("text_encoder.")}
        if te and config.text_encoder:
            from transformers import AutoConfig, AutoModelForTextEncoding
            tcfg = dict(config.text_encoder)
            tc = AutoConfig.for_model(tcfg.pop("model_type"), **tcfg)
            text_encoder = AutoModelForTextEncoding.from_config(tc)
            text_encoder.load_state_dict(te, strict=False)
            text_encoder = text_encoder.to(device=device, dtype=torch_dtype).eval()
        m = cls(config, device=device, dtype=torch_dtype, text_encoder=text_encoder)
        m.load_state_dict(sd)
        gpath = os.path.join(path, "generation_config.json")
        if os.path.exists(gpath):
            with open(gpath) as f:
                m.generation_config.update(**json.load(f))
        return m

    def to(self, *a, **k):
        return self

    def eval(self):
        return self

    # -- side inputs (not replaced; PyTorch) -------------------------------------------------------
    def _encode_text_eager(self, input_ids, attention_mask, flags: Optional[dict] = None):
        """flags: None, or output_attentions / output_hidden_states for the encoder: then (states, the encoder's output)."""
        enc_mask = attention_mask
        if attention_mask is not None and attention_mask.dim() == 2:
            # the 4-D additive form HF derives from a 2-D padding mask (0 keep / finfo.min drop), built here with device ops only:
            # the library's own conversion creates CPU scalars on the way, which a CUDA-graph capture cannot contain
            edt = next(self.text_encoder.parameters()).dtype
            enc_mask = (1 - attention_mask)[:, None, None, :].to(edt) * torch.finfo(edt).min
        eo = self.text_encoder(input_ids=input_ids, attention_mask=enc_mask, return_dict=True, **(flags or {}))
        h = eo.last_hidden_state
        if self.enc_to_dec_proj is not None:
            h = torch.nn.functional.linear(h, *self.enc_to_dec_proj)        # :2388-2392 / :3087-3090
        if attention_mask is not None:
            h = h * attention_mask[..., None]                               # :3092-3093
        return h.to(self.dtype) if flags is None else (h.to(self.dtype), eo)

    def _encode_text(self, input_ids, attention_mask):
        """Description ids -> encoder_hidden_states (reference :3048-3097): T5 encoder + enc_to_dec_proj + mask multiply.
        These PyTorch modules are not replaced (SURVEY section 8 f3); what this path adds is ONE CUDA graph per (batch, length) shape
        over the whole chain -- a T5 encoder is ~150 small launches whose launch latency, not their math, is the time-to-first-audio
        once the decode loop is fast.  Inputs are copied into static buffers and the graph is replayed; if capture is impossible
        (a module that synchronises), the eager path is used and said so once."""
        if self.text_encoder is None:
            raise ValueError("this model was built without a text encoder: pass `encoder_outputs`")
        input_ids = input_ids.to(self.device)
        attention_mask = None if attention_mask is None else attention_mask.to(self.device)
        if not hasattr(self, "_enc_graphs"):
            self._enc_graphs, self._enc_graph_ok = {}, True
        if not self._enc_graph_ok or self.device.type != "cuda":
            return self._encode_text_eager(input_ids, attention_mask)
        key = (tuple(input_ids.shape), attention_mask is not None)
        entry = self._enc_graphs.get(key)
        if entry is None:
            try:
                s_ids = input_ids.clone()
                s_mask = None if attention_mask is None else attention_mask.clone()
                side = torch.cuda.Stream(device=self.device)
                side.wait_stream(torch.cuda.current_stream(self.device))
                with torch.cuda.stream(side):
                    for _ in range(2):                                   # warm-up: lazy initialisations happen outside the capture
                        self._encode_text_eager(s_ids, s_mask)
                torch.cuda.current_stream(self.device).wait_stream(side)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    s_out = self._encode_text_eager(s_ids, s_mask)
                entry = (graph, s_ids, s_mask, s_out)
                if len(self._enc_graphs) >= 16:
                    self._enc_graphs.clear()
                self._enc_graphs[key] = entry
            except Exception as ex:  # pragma: no cover - depends on the encoder implementation
                import warnings
                warnings.warn(f"text-encoder CUDA graph capture failed ({ex!r}); running the encoder eagerly")
                self._enc_graph_ok = False
                torch.cuda.synchronize(self.device)
                return self._encode_text_eager(input_ids, attention_mask)
        graph, s_ids, s_mask, s_out = entry
        s_ids.copy_(input_ids)
        if s_mask is not None:
            s_mask.copy_(attention_mask)
        graph.replay()
        return s_out.clone()

    # -- conditioning (forward and generate) --------------------------------------------------------
    def _conditioning(self, caller: str, input_ids, attention_mask, encoder_outputs, prompt_input_ids, prompt_attention_mask,
                      prompt_hidden_states, cross_prompt_after_encoder_outputs: bool, encoder_flags: Optional[dict] = None):
        """forward()'s and generate()'s inputs -> (encoder states [B, S, H], their mask, the prompt prefix [B, P, H] or None, its
        mask, the transcript keys as (first key, count, mask), the text encoder's output if encoder_flags ran it eagerly, else None).
        On a prompt_cross_attention checkpoint the prompt joins the description as cross-attention keys (prompt_cross_states,
        :2791-2811 / :3099-3130) and there is no prefix; with `encoder_outputs` only if cross_prompt_after_encoder_outputs."""
        cross_prompt = self.prompt_cross_attention and (prompt_input_ids is not None or prompt_hidden_states is not None)
        eo = None
        if encoder_outputs is not None:
            if cross_prompt and not cross_prompt_after_encoder_outputs:
                # the reference would make the prompt a self-attention prefix without positions: the other model
                raise ValueError("a prompt_cross_attention model joins the prompt to the description only when forward() runs the "
                                 "text encoder: pass `input_ids` instead of `encoder_outputs`, or no prompt")
            enc = encoder_outputs
            enc_hidden = enc[0] if isinstance(enc, (tuple, list)) else getattr(enc, "last_hidden_state", enc)
        elif input_ids is None:
            raise ValueError(f"{caller}() needs `input_ids` (description) or `encoder_outputs`")
        elif encoder_flags:
            enc_hidden, eo = self._encode_text_eager(input_ids, attention_mask, encoder_flags)
        else:
            enc_hidden = self._encode_text(input_ids, attention_mask)   # encoder + enc_to_dec_proj + mask multiply, one CUDA graph
        enc_hidden = enc_hidden.to(self.device, self.dtype)
        if cross_prompt:
            prompt = prompt_hidden_states if prompt_hidden_states is not None else prompt_input_ids
            if prompt.dim() == 2 and not self._side_loaded:
                raise ValueError("no embed_prompts weights loaded")
            text = (enc_hidden.shape[1], prompt.shape[1], prompt_attention_mask)
            enc_hidden, attention_mask = prompt_cross_states(enc_hidden, attention_mask, prompt, prompt_attention_mask,
                                                             self.embed_prompts_weight, self.embed_positions_weight)
            return enc_hidden, attention_mask, None, None, text, eo
        prompt_hidden = prompt_hidden_states
        if prompt_hidden is None and prompt_input_ids is not None:
            if not self._side_loaded:
                raise ValueError("no embed_prompts weights loaded")
            prompt_hidden = torch.nn.functional.embedding(prompt_input_ids.to(self.device), self.embed_prompts_weight)
        prompt_mask = prompt_attention_mask if prompt_hidden is not None else None
        text = (0, 0 if prompt_hidden is None else prompt_hidden.shape[1], prompt_mask)
        return enc_hidden, attention_mask, prompt_hidden, prompt_mask, text, eo

    def _encode_clips(self, clips, B: int):
        """generate(input_values=[w_0, ..]): each clip [1, samples_b] or [samples_b] through one ragged DACModel.encode call
        (the clips right-padded to the longest, sample_lengths = their lengths) -> the codes right-padded to the longest,
        [B, K, N_max] with 0 past each clip's frames, and their frame mask [B, N_max]."""
        K = self.config.decoder.num_codebooks
        if len(clips) != B:
            raise ValueError(f"input_values must hold batch_size = {B} clips, got {len(clips)}")
        if self.config.audio_encoder.num_codebooks != K:
            raise ValueError(f"the codec has {self.config.audio_encoder.num_codebooks} codebooks, the decoder {K}: "
                             "its codes cannot continue this decoder")
        wavs = []
        for i, w in enumerate(clips):
            w = torch.as_tensor(w)
            if w.dim() == 2 and w.shape[0] == 1:
                w = w[0]
            if w.dim() != 1 or w.shape[0] < 1:
                raise ValueError(f"input_values[{i}] must be [1, samples] or [samples], got {tuple(w.shape)}")
            wavs.append(w)
        for i, w in enumerate(wavs):
            if not w.is_floating_point():
                raise ValueError(f"input_values[{i}] must be a floating-point waveform, got {w.dtype}")
        # one dtype every clip widens to exactly, so that each is rounded to the model dtype as it would be on its own
        dtype = functools.reduce(torch.promote_types, [w.dtype for w in wavs])
        lens = [w.shape[0] for w in wavs]
        wav = torch.zeros(B, max(lens), dtype=dtype, device=self.device)
        for i, w in enumerate(wavs):
            wav[i, :lens[i]] = w.to(self.device)
        codes = self.audio_encoder.encode(wav[:, None, :], sample_lengths=lens).audio_codes.reshape(B, K, -1)
        hop = self.audio_encoder.hop_length
        frames = torch.tensor([-(-n // hop) for n in lens])
        mask = (torch.arange(codes.shape[-1])[None, :] < frames[:, None]).to(torch.int64)
        ids = codes.masked_fill(mask.to(self.device)[:, None, :] == 0, 0)
        return ids, mask

    def _codes_from_raw(self, output_ids, mask_src, max_length: int):
        """The raw token matrix [B * K, T] of one decoder input mask_src [B * K, n0] -> (the de-delayed matrix, codes [B, K, F])."""
        d = self.config.decoder
        K = d.num_codebooks
        _, full_mask = build_delay_pattern_mask(mask_src, d.bos_token_id, d.pad_token_id, max_length, K)
        output_ids = apply_delay_pattern_mask(output_ids, full_mask)
        _, mask = build_delay_pattern_mask(mask_src, d.bos_token_id, d.pad_token_id, output_ids.shape[1], K)
        keep = (mask != d.bos_token_id) & (mask != d.pad_token_id)
        return output_ids, output_ids[keep].reshape(output_ids.shape[0] // K, K, -1)

    def _ragged_codes_from_raw(self, output_ids, dec_ids, input_lens, max_length: int):
        """A ragged continuation's raw token matrix [B * K, T] -> (de-delayed matrix, codes [B, K, F_max]).  Row b holds its own
        columns [0, T - s_b) with s_b = n0 - n0_b, and gets its own delay pattern (its input's first n0_b columns, max_length - s_b),
        what the row alone would get; past its columns (and its frames in `codes`) the rows are filled with pad_token_id."""
        d = self.config.decoder
        K, T, n0 = d.num_codebooks, output_ids.shape[1], dec_ids.shape[1]
        B = output_ids.shape[0] // K
        shift = (n0 - input_lens).cpu()
        out = torch.full_like(output_ids, d.pad_token_id)
        rows_codes = [None] * B
        for s in sorted(set(shift.tolist())):
            idx = torch.nonzero(shift == s).flatten()
            rows = (idx[:, None] * K + torch.arange(K)[None, :]).flatten().to(output_ids.device)
            o, c = self._codes_from_raw(output_ids[rows, :T - s].contiguous(), dec_ids[rows, :n0 - s].contiguous(), max_length - s)
            out[rows, :T - s] = o
            for j, b in enumerate(idx.tolist()):
                rows_codes[b] = c[j]
        F = max(c.shape[-1] for c in rows_codes)
        codes = torch.full((B, K, F), d.pad_token_id, dtype=torch.int64, device=output_ids.device)
        for b, c in enumerate(rows_codes):
            codes[b, :, :c.shape[-1]] = c
        return out, codes

    # -- the token loop ------------------------------------------------------------------------------
    def _sampling(self, gc, n0: int, max_length: int, seed=0, suppress_special=False, row_base=0, logits_processor=None,
                  stopping_criteria=None) -> Sampling:
        """A generate() call's Sampling for n0 decoder input columns; resolve_sampling_ext / resolve_logits_ext raise here."""
        d = self.config.decoder
        ext, min_new_tokens = resolve_sampling_ext(gc, n0)
        lext = resolve_logits_ext(gc, n0, max_length, d.vocab_size, d.eos_token_id)
        return Sampling(max_length, gc.do_sample, gc.temperature, gc.top_k if gc.do_sample else 0, gc.top_p, min_new_tokens, seed,
                        suppress_special, self.config.audio_encoder.codebook_size, row_base, ext, lext, list(logits_processor or []),
                        list(stopping_criteria or []))

    def _host_driven_loop(self, sess: "GenSession", s: Sampling, streamer, stream_col, outputs, out_row, window):
        """One host iteration per token, like GenerationMixin._sample: the decoder step still runs on the fused kernel
        (ptts_decode_forward), the built-in processors run as their device operators (MinNewTokens as a mask,
        ParlerTTSLogitsProcessor = ptts_logits_processor), then the caller's `logits_processor` list, the HF warpers and the draw
        as torch ops on the device scores, and the token is appended with ptts_sample(forced).  Used only when the caller passes
        processors or criteria the device loop does not know (the reference merges such lists at :3540-3552).  `s.ext`
        (resolve_sampling_ext) adds the n-gram bans before the EOS masks and the MinP / Typical / Epsilon / Eta warpers after
        top-p, in transformers' order; `s.lext` (resolve_logits_ext) adds sequence_bias first, forced BOS / EOS, InfNan, the decay
        and the suppress lists before the Parler EOS processor, and LogitNormalization last (greedy's argmax and the draw use the
        scores before it, as the device loop does).  `outputs` (StepOutputs) records each step's raw logits and final scores
        before the draw, from row out_row on; `window(step)` attaches the other recorders before each decoder step."""
        d = self.config.decoder
        K, BK = d.num_codebooks, sess.B * d.num_codebooks
        ext, lext = s.ext, s.lext
        parler = ParlerTTSLogitsProcessor(d.eos_token_id, K, sess.B, self.device)
        gen = torch.Generator(device=self.device).manual_seed(int(s.seed))
        unfinished = torch.ones(BK, dtype=torch.long, device=self.device)
        cur = sess.n0   # the first new column follows the decoder input (the BOS column, or BOS + code prefix)
        while True:
            ids = sess.raw_ids[:, :cur]
            scores = sess.logits.clone()
            if lext is not None:
                scores = lext.sequence_bias(ids, scores)
            if ext is not None:
                scores = no_repeat_ngram_mask(ids, scores, ext["no_repeat_ngram_size"])
            if s.min_new_tokens > 0 and cur - sess.n0 < s.min_new_tokens:
                scores[:, d.eos_token_id] = -float("inf")
            if lext is not None:
                scores = lext.before_parler(ids, scores).contiguous()
            scores = parler(ids, scores)
            for proc in s.processors:
                scores = proc(ids, scores)
            if s.do_sample:
                if s.temperature and s.temperature != 1.0:
                    scores = scores / s.temperature
                if s.top_k:
                    kth = torch.topk(scores, min(int(s.top_k), scores.shape[-1]))[0][..., -1, None]
                    scores = scores.masked_fill(scores < kth, -float("inf"))
                if s.top_p is not None and s.top_p < 1.0:
                    ss, si = torch.sort(scores, descending=False)
                    rem = ss.softmax(-1).cumsum(-1) <= (1 - s.top_p)
                    rem[..., -1:] = False
                    scores = scores.masked_fill(rem.scatter(1, si, rem), -float("inf"))
                if ext is not None:
                    scores = sampling_ext_warpers(scores, ext)
            final = scores if lext is None else lext.normalize(scores)   # what transformers' _sample records and passes on
            if outputs is not None:
                outputs.put(cur - sess.n0, out_row, sess.logits, final)
            if s.do_sample:
                nxt = torch.multinomial(scores.softmax(-1), 1, generator=gen).squeeze(1)
            else:
                nxt = scores.argmax(-1)
            nxt = nxt * unfinished + d.pad_token_id * (1 - unfinished)
            sess.sample(forced=nxt)           # append (+ delay-pattern override of the next input), device-side stopping state
            if streamer is not None:
                streamer.put(stream_col(cur, nxt).cpu())
            cur += 1
            unfinished = unfinished & ~((nxt == d.eos_token_id) | (cur >= s.max_length)).long()
            stop = unfinished.max().item() == 0
            for crit in s.criteria:
                r = crit(sess.raw_ids[:, :cur], final)
                r = r if isinstance(r, torch.Tensor) else torch.full((BK,), bool(r), device=self.device)
                unfinished = unfinished & ~r.long()
                stop = stop or unfinished.max().item() == 0
            if stop:
                break
            window(cur - sess.n0)
            sess.decode_forward()

    def _fused_batch_limit(self):
        """Rows one fused decode-step launch covers (None: the fused kernels are not in play, the batch runs as one session)."""
        if self.dtype != torch.bfloat16 or os.environ.get("PTTS_FUSED", "1") == "0":
            return None
        return 32

    def _run_token_loop(self, enc_hidden, enc_mask, prompt_hidden, prompt_mask, input_ids, sampling: Sampling, shard, recorders=(),
                        streamer=None, input_lens=None):
        """begin + prefill + the token loop of one shard's session -> its raw token matrix [rows * K, generated length].
        The inputs are the whole call's: enc_hidden / enc_mask per description, prompt_hidden / prompt_mask per take, input_ids
        None or the BOS-led decoder input [takes * K, n0], input_lens None or each take's own column count [takes] (a ragged
        continuation; the shard passes its slice, or None when all of it is n0).  shard: (first description, end, first take,
        end) (take_shards).
        recorders (see recording): the device loop keeps each decode_steps call inside one chunk of those that have chunks."""
        d = self.config.decoder
        K, s = d.num_codebooks, sampling
        d0, d1, r0, r1 = shard
        cut = lambda t, a, b: None if t is None else t[a:b]
        enc_hidden, enc_mask = enc_hidden[d0:d1], cut(enc_mask, d0, d1)
        prompt_hidden, prompt_mask, input_ids = cut(prompt_hidden, r0, r1), cut(prompt_mask, r0, r1), cut(input_ids, r0 * K, r1 * K)
        B, S = r1 - r0, enc_hidden.shape[1]
        P = 0 if prompt_hidden is None else prompt_hidden.shape[1]
        n0 = 1 if input_ids is None else int(input_ids.shape[1])
        input_lens = cut(input_lens, r0, r1)
        if input_lens is not None and bool((input_lens == n0).all()):
            input_lens = None
        sess = self.decoder.engine.session(B, P, S, P + s.max_length, max_input_len=n0, takes=B // (d1 - d0))
        host = bool(s.processors or s.criteria)
        sess.begin(s.max_length, do_sample=s.do_sample, temperature=s.temperature, top_k=s.top_k, top_p=s.top_p,
                   min_new_tokens=s.min_new_tokens, seed=s.seed, suppress_special=s.suppress_special, codebook_size=s.codebook_size,
                   row_base=s.row_base + r0 * K, input_ids=input_ids, input_lens=input_lens,
                   ext=None if host else s.ext, lext=None if host else s.lext)    # the host-driven loop applies them as torch ops
        stream_col = lambda col, v: v
        if streamer is not None:
            if input_ids is None:
                streamer.put(torch.full((B * K, 1), d.bos_token_id, dtype=torch.int64))
            else:
                streamer.put(sess.raw_ids[:, :n0].cpu())   # the whole delayed input first (:3534)
                # Codebook k's prefix ids reach K-1 columns past the delayed input; generate()'s result takes them there
                # (the pattern mask, :3586), so the streamed columns carry them too.
                _, pm = build_delay_pattern_mask(input_ids, d.bos_token_id, d.pad_token_id, s.max_length, K)
                cells = pm[:, n0:n0 + K - 1]
                stream_col = lambda col, v: (torch.where(cells[:, col - n0] == -1, v, cells[:, col - n0]) if col - n0 < cells.shape[1] else v)
        # The host-driven loop draws the token in torch and copies the outputs from there (StepOutputs.put): the sampler records
        # none, so only the other recorders get windows.
        outputs = next((r for r in recorders if isinstance(r, StepOutputs)), None) if host else None
        windows = [r for r in recorders if r is not outputs]

        def window(step):
            for r in windows:
                r.attach_window(sess, step, r0)
        with recording(sess, recorders, r0):
            sess.prefill(prompt_hidden, prompt_mask, enc_hidden, enc_mask)
            if host:
                self._host_driven_loop(sess, s, streamer, stream_col, outputs, r0 * K, window)
            else:
                window(0)
                sess.sample()
                step, steps_left = 1, s.max_length - n0 - 1
                chunked = any(r.CHUNK for r in windows)
                if streamer is not None:
                    streamer.put(stream_col(n0, sess.raw_ids[:, n0]).cpu())
                # Without a streamer there is no per-step host sync: decode_steps enqueues up to 64 tokens (one cluster kernel
                # launch) and the device `active` flag is read between calls.  A streamer gets one host-visible column per step
                # (_sample -> streamer.put(next.cpu())), and none after the session went inactive.
                while steps_left > 0:
                    if streamer is not None and int(sess.state[1].item()) != 1:
                        break
                    n = 1 if streamer is not None else steps_in_window(step, steps_left, StepOutputs.CHUNK) if chunked else min(64, steps_left)
                    window(step)
                    sess.decode_steps(n)
                    step, steps_left = step + n, steps_left - n
                    if streamer is not None:
                        streamer.put(stream_col(n0 + step - 1, sess.raw_ids[:, n0 + step - 1]).cpu())
                    elif steps_left > 0 and int(sess.state[1].item()) == 0:
                        break
            if streamer is not None:
                streamer.end()
        cur_len = int(sess.state[0].item())
        return sess.raw_ids[:, :cur_len].clone()

    def _token_timestamps(self, align: StepAlignment, raw_ids: torch.Tensor, n0: int, text_mask, takes: int) -> dict:
        """generate()'s `alignment` [B * N, T_gen, P] and `token_timestamps` [B * N, P] (seconds from the first generated frame,
        NaN at masked transcript positions): the recorded rows, then ptts_align_dtw over each utterance's token_frames."""
        K, cs = self.config.decoder.num_codebooks, self.config.audio_encoder.codebook_size
        alignment = align.alignment[:, :raw_ids.shape[1] - n0].contiguous()
        mask = None
        if text_mask is not None:
            mask = text_mask.to(self.device)
            if mask.shape[0] != alignment.shape[0]:
                mask = mask.repeat_interleave(takes, dim=0)
        _, jumps = align_dtw(alignment, token_frames(raw_ids, n0, K, cs), mask)
        seconds = jumps.double() * self.audio_encoder.hop_length / self.config.audio_encoder.sampling_rate
        return dict(alignment=alignment, token_timestamps=torch.where(jumps >= 0, seconds, float("nan")).float())

    # -- teacher-forced forward (scoring) ------------------------------------------------------------
    _SCORE_SHARD = 32   # utterances per ptts_score call: the workspace is sized for one shard

    @torch.no_grad()
    def forward(self, input_ids=None, attention_mask=None, input_values=None, padding_mask=None, decoder_input_ids=None,
                decoder_attention_mask=None, encoder_outputs=None, prompt_input_ids=None, prompt_attention_mask=None,
                prompt_hidden_states=None, labels=None, loss_reduction: str = "mean", return_logits: bool = False,
                output_attentions: bool = False, output_hidden_states: bool = False, **kwargs):
        """The reference's model call (:2695-2880) for inference-time scoring: the decoder over the prompt prefix and the T decoder
        input columns in one prefill pass, the K lm heads over the T positions, and the loss of :1922-1974.

        labels [B, T, K] (training format: delayed, -100 where ignored) give decoder_input_ids = shift_tokens_right(labels)
        .transpose(1, 2) unless decoder_input_ids are passed ([B * K, T] or [B, K, T], used as given).  loss_reduction is "mean"
        or "sum"; config.decoder.codebook_weights weight the codebooks as in the reference.  Returns a ParlerTTSSeq2SeqLMOutput
        with loss, per_codebook_losses and token_losses [B, T, K] (the NLL of each counted label, 0 elsewhere: what a reranker
        sums per utterance).  One deviation: with labels, `logits` [B * K, T, V] is filled only if return_logits=True (otherwise
        None), because the fused kernel exists so that tensor (0.5-3 GB) is never built; without labels it is always filled.
        decoder_attention_mask must be right padding, which changes nothing the loss keeps under the causal mask.  Training
        (backward) is out of scope.

        output_attentions / output_hidden_states add decoder_attentions (L x [B, heads, P+T, P+T]), cross_attentions
        (L x [B, heads, P+T, S]) and decoder_hidden_states (L+1 x [B, P+T, H]) in the model dtype, written by the same pass (the
        weights by the reference's eager definition, see generate()); the loss, token_losses and logits do not change.

        config.prompt_cross_attention: when forward() runs the text encoder, `prompt_input_ids` or `prompt_hidden_states` plus
        their positions join the description as cross-attention keys (prompt_cross_states, :2791-2811) and P = 0; with
        `encoder_outputs` a prompt raises ValueError."""
        if kwargs:
            raise ValueError(f"forward() got arguments this path does not take: {sorted(kwargs)}")
        if loss_reduction not in ("mean", "sum"):
            raise ValueError(f"loss_reduction must be 'mean' or 'sum', got {loss_reduction!r}")
        if labels is None and decoder_input_ids is None:
            if input_values is not None:
                raise ValueError("forward(input_values=...) without labels or decoder_input_ids: encode the audio with "
                                 "audio_encoder.encode(...) and pass its codes as decoder_input_ids")
            raise ValueError("forward() needs `labels` or `decoder_input_ids`")
        enc_hidden, attention_mask, prompt_hidden, prompt_mask, _, _ = self._conditioning(
            "forward", input_ids, attention_mask, encoder_outputs, prompt_input_ids, prompt_attention_mask, prompt_hidden_states,
            cross_prompt_after_encoder_outputs=False)
        if enc_hidden.dim() != 3 or enc_hidden.shape[2] != self.config.decoder.hidden_size:
            raise ValueError(f"encoder states must be [batch, length, {self.config.decoder.hidden_size}], got {tuple(enc_hidden.shape)}")
        B, S, _ = enc_hidden.shape
        if attention_mask is not None and tuple(attention_mask.shape) != (B, S):
            raise ValueError(f"attention_mask must be [{B}, {S}], got {tuple(attention_mask.shape)}")
        P = 0 if prompt_hidden is None else prompt_hidden.shape[1]
        if prompt_hidden is not None and (prompt_hidden.dim() != 3 or prompt_hidden.shape[0] != B):
            raise ValueError(f"prompt states must be [{B}, P, H], got {tuple(prompt_hidden.shape)}")
        if prompt_mask is not None and tuple(prompt_mask.shape) != (B, P):
            raise ValueError(f"prompt_attention_mask must be [{B}, {P}], got {tuple(prompt_mask.shape)}")
        d = self.config.decoder
        K, V = d.num_codebooks, d.vocab_size
        labels, dec = check_scoring_inputs(labels, decoder_input_ids, decoder_attention_mask, batch_size=B, num_codebooks=K,
                                           vocab_size=V, pad_token_id=self.config.pad_token_id,   # the top-level ids, as :2821
                                           decoder_start_token_id=self.config.decoder_start_token_id, prompt_len=P,
                                           max_position_embeddings=d.max_position_embeddings)
        T = dec.shape[1]
        dev = self.device
        want_logits = labels is None or bool(return_logits)
        token_nll = None if labels is None else torch.empty(B, T, K, dtype=torch.float32, device=dev)
        logits = torch.empty(B * K, T, V, dtype=torch.float32, device=dev) if want_logits else None
        n_shards = (B + self._SCORE_SHARD - 1) // self._SCORE_SHARD
        sums = None if labels is None else torch.empty(n_shards, K, 2, dtype=torch.float32, device=dev)
        cut = lambda t, sl: None if t is None else t[sl]
        probes = None
        if output_attentions or output_hidden_states:
            probes = StepProbes(d.num_hidden_layers, B, d.num_attention_heads, S, d.hidden_size, P, T, self.dtype, dev,
                                output_attentions, output_hidden_states)
        for i, b0 in enumerate(range(0, B, self._SCORE_SHARD)):
            sl = slice(b0, min(B, b0 + self._SCORE_SHARD))
            sess = self.decoder.engine.session(sl.stop - sl.start, P, S, P + T, max_input_len=T)
            with recording(sess, [] if probes is None else [probes], b0):
                sess.score(cut(prompt_hidden, sl), cut(prompt_mask, sl), enc_hidden[sl], cut(attention_mask, sl),
                           dec[sl.start * K:sl.stop * K], cut(labels, sl), cut(token_nll, sl),
                           None if logits is None else logits[sl.start * K:sl.stop * K], None if sums is None else sums[i])
        loss = per_codebook = None
        if labels is not None:
            # per codebook: sum (and count) over the shards, then the reference's reduction; a mean over no cell is NaN as in torch
            tot = sums.double().sum(0)
            per = tot[:, 0] / tot[:, 1] if loss_reduction == "mean" else tot[:, 0]
            w = d.codebook_weights
            if w is not None:
                wt = torch.tensor([float(x) for x in w], dtype=torch.float64, device=dev)
                loss = ((per * wt).sum() / wt.sum()).float()
            else:
                loss = (per.sum() / K).float()
            per_codebook = [per[k].float() for k in range(K)]
        out = ParlerTTSSeq2SeqLMOutput(loss=loss, logits=logits, per_codebook_losses=per_codebook, token_losses=token_nll,
                                       encoder_last_hidden_state=enc_hidden)
        if probes is not None:
            out.update(probes.entry(0))
        return out

    __call__ = forward

    # -- generate ----------------------------------------------------------------------------------
    @torch.no_grad()
    def generate(self, inputs: Optional[torch.Tensor] = None, generation_config: Optional[GenerationConfig] = None,
                 logits_processor=None, stopping_criteria=None, synced_gpus=None, streamer=None, **kwargs):
        """Same call contract as the reference generate() (:3322-3653) for greedy / sampling modes.

        Extra kwargs: `seed` (Philox key for sampling, default 0), `return_codes` (also return audio codes).

        With return_dict_in_generate=True, output_scores / output_logits add `scores` / `logits` as in transformers' _sample: a
        tuple with one fp32 [B * K, V] entry per generated column (column n0 + t was drawn from entry t), the processed scores the
        token was drawn from (-inf where removed) and the raw logits.  Rows that finished keep being recorded while the session
        runs.  Deviation: a batch above 32 utterances runs as shards of 32, and a shard that ended holds NaN in both up to the
        longest shard's end.

        output_attentions / output_hidden_states (with return_dict_in_generate=True) add transformers' `decoder_attentions`,
        `cross_attentions` and `decoder_hidden_states`, one entry per generated column indexed like `scores`: entry 0 is the
        prefill (q = P + n0 rows: the prompt prefix, then BOS or the code prefix), entry t >= 1 has q = 1 and T_kv = P + n0 + t
        keys.  Attention entries are tuples of L [B, heads, q, T_kv] (cross: [B, heads, q, S]) tensors, hidden-state entries
        tuples of L + 1 [B, q, H] (the embeddings, the outputs of layers 0 .. L-2, the final LayerNorm of the last layer's output),
        all in the model dtype.  When generate() runs the text encoder itself, `encoder_attentions` / `encoder_hidden_states`
        come from an eager call of it with the same flags (None with `encoder_outputs`).  The weights follow the reference's eager
        attention (model-dtype scores, fp32 softmax), computed from the q and K the session holds.  Deviations: in the reference,
        asking for attentions switches its own attention to that eager path and can change its tokens; here the tokens, scores
        and audio are bit-identical with and without the flags, while the decode steps run the multi-kernel path (not the fused
        step kernel) for as long as anything is recorded.  A shard that ended holds NaN, as in `scores`.  Memory: see
        StepProbes.

        return_token_timestamps=True (with return_dict_in_generate=True, else ValueError) adds `alignment` [B * N, T_gen, P] fp32,
        row t the mean over `alignment_heads` ([layer, head] pairs; None = every head of the last ceil(L / 2) layers) of each
        head's weights over the P transcript tokens, renormalized over them (masked tokens 0), for the query of generated column
        n0 + t (the last row, never a decode step's input, is NaN), and `token_timestamps` [B * N, P] fp32: each transcript
        token's start in seconds, counted from the first generated frame (after a continuation's prefix audio), NaN where the
        prompt is masked (StepAlignment, align_dtw).  The transcript is the prompt prefix, or the prompt's cross-attention keys
        in prompt_cross_attention mode; without one the flag raises ValueError.  The tokens and audio do not change; the decode
        steps run the multi-kernel path while it is set.

        config.prompt_cross_attention: `prompt_input_ids` plus their sinusoidal positions are appended to the description states
        as cross-attention keys (prompt_cross_states, reference :3099-3130), also after `encoder_outputs`; the decoder then has no
        prompt prefix (P = 0), and `cross_attentions` have S + P keys.  `prompt_hidden_states` raise ValueError in this mode.

        num_return_sequences = N (an int >= 1; > 1 needs do_sample=True, as in transformers) draws N takes per description: every
        per-utterance output has B * N rows, take n of description b at row b * N + n (`sequences`, `audio_codes`, `audios_length`,
        `raw_ids`, the streamer's rows, the [B * N * K, V] `scores` / `logits` entries, the batch index of the decoder probes), and
        it draws exactly what row b * N + n of the hand-expanded batch would (Philox substream (b * N + n) * K + k + row_base).  The
        text encoder runs once per description (`encoder_attentions` / `encoder_hidden_states` stay B-sized) and the takes of a
        description share one copy of its cross-attention K/V; a self-attention prompt prefix and a continuation's codes
        (`decoder_input_ids` / `input_values`, encoded once) are repeated per take, as one group of K code rows per utterance.
        """
        import copy
        gc = copy.deepcopy(generation_config if generation_config is not None else self.generation_config)
        seed = kwargs.pop("seed", 0)
        row_base = kwargs.pop("row_base", 0)   # batch shards: global (utterance x codebook) row of this shard's first row (dist.py)
        return_codes = kwargs.pop("return_codes", False)
        suppress_special = kwargs.pop("_suppress_special", False)
        user_max_length = kwargs.get("max_length")
        mk = gc.update(**kwargs)
        # The reference would honour (or reject) every generation knob; silently dropping one changes the output without an error.
        unknown = sorted(k for k in mk if k not in self._MODEL_KWARGS)
        if unknown:
            raise ValueError(f"The following `model_kwargs` are not used by the model: {unknown} (note: typos in the generate "
                             "arguments will also show up in this list)")
        for k in ("use_cache", "cache_implementation"):
            mk.pop(k, None)   # accepted for call compatibility: the device loop always uses its static cache
        unsupported = {k: getattr(gc, k) for k, neutral in self._NEUTRAL_GENERATION_KNOBS.items() if getattr(gc, k, neutral) != neutral}
        if unsupported:
            raise ValueError(f"generation options {unsupported} are not supported by the device loop (greedy / sampling with "
                             "temperature, top_k, top_p, min_p, typical_p, epsilon_cutoff, eta_cutoff, no_repeat_ngram_size, "
                             "min_length, min_new_tokens, sequence_bias, suppress_tokens, begin_suppress_tokens, "
                             "exponential_decay_length_penalty, forced_bos_token_id, forced_eos_token_id, remove_invalid_values and "
                             "renormalize_logits only)")
        if gc.num_beams != 1:
            raise ValueError("Got incompatible mode for generation, should be one of greedy or sampling. "
                             "Ensure that beam search is de-activated by setting `num_beams=1` and `num_beam_groups=1`.")
        N = resolve_num_return_sequences(gc)
        want_ts = bool(gc.return_token_timestamps)
        if want_ts and not gc.return_dict_in_generate:
            raise ValueError("`return_token_timestamps=True` needs `return_dict_in_generate=True`: the alignment and the "
                             "timestamps exist only in the dict return")
        align_heads = None
        if want_ts or gc.alignment_heads is not None:
            align_heads = resolve_alignment_heads(gc.alignment_heads, self.config.decoder.num_hidden_layers,
                                                  self.config.decoder.num_attention_heads)
        if self.prompt_cross_attention and mk.get("prompt_hidden_states") is not None:
            # the reference would put these states in front of the decoder while counting its cache positions without them
            raise ValueError("a prompt_cross_attention model takes the transcript as `prompt_input_ids`, not `prompt_hidden_states`")
        # decoder_attentions / cross_attentions / decoder_hidden_states exist only in the dict return, as in transformers
        want_attn = bool(gc.return_dict_in_generate and gc.output_attentions)
        want_hidden = bool(gc.return_dict_in_generate and gc.output_hidden_states)
        enc_hidden, attention_mask, prompt_hidden, prompt_mask, (text_key0, text_len, text_mask), eo = self._conditioning(
            "generate", mk.get("input_ids", inputs), mk.get("attention_mask"), mk.get("encoder_outputs"), mk.get("prompt_input_ids"),
            mk.get("prompt_attention_mask"), mk.get("prompt_hidden_states"), cross_prompt_after_encoder_outputs=True,
            # the encoder's own tuples: one eager call with the flags
            encoder_flags=dict(output_attentions=want_attn, output_hidden_states=want_hidden) if want_attn or want_hidden else None)
        P = 0 if prompt_hidden is None else prompt_hidden.shape[1]
        B, S, _ = enc_hidden.shape
        if want_ts and text_len == 0:
            raise ValueError("`return_token_timestamps=True` needs a transcript to align: pass `prompt_input_ids` or "
                             "`prompt_hidden_states` with at least one token")

        d = self.config.decoder
        K = d.num_codebooks
        dec_ids = input_lens = None
        # code prefixes of different lengths: a decoder_attention_mask, or the clips of a list of input_values (ragged mode)
        ragged = mk.get("decoder_attention_mask") is not None or (mk.get("decoder_input_ids") is None and
                                                                  isinstance(mk.get("input_values"), (list, tuple)))
        if ragged:
            check_ragged_generate(streamer, logits_processor, stopping_criteria, gc)
            if mk.get("decoder_input_ids") is None and mk.get("input_values") is None:
                raise ValueError("decoder_attention_mask needs decoder_input_ids (or input_values) to apply to")
        if mk.get("decoder_input_ids") is None and isinstance(mk.get("input_values"), (list, tuple)):
            mk["decoder_input_ids"], mk["decoder_attention_mask"] = self._encode_clips(mk["input_values"], B)
        elif mk.get("decoder_input_ids") is None and mk.get("input_values") is not None:
            # audio prompt (:3442-3446, :3136-3194): encoded once, with every codebook; its codes continue like decoder_input_ids.
            # padding_mask does not reach the encoder, as in the reference.
            wav = mk["input_values"]
            if wav.dim() != 3 or wav.shape[0] != B:
                raise ValueError(f"input_values must be [batch_size = {B}, 1, samples], got {tuple(wav.shape)}")
            if self.config.audio_encoder.num_codebooks != K:
                raise ValueError(f"the codec has {self.config.audio_encoder.num_codebooks} codebooks, the decoder {K}: "
                                 "its codes cannot continue this decoder")
            mk["decoder_input_ids"] = self.audio_encoder.encode(wav).audio_codes
        if mk.get("decoder_input_ids") is not None:   # -> the BOS-led [B * K, n0] on the device (:3012-3024)
            start = gc.decoder_start_token_id if gc.decoder_start_token_id is not None else d.bos_token_id
            if ragged:   # + each row's own column count n0_b
                dec_ids, input_lens = prepare_ragged_decoder_input_ids(mk["decoder_input_ids"], mk["decoder_attention_mask"], B, K,
                                                                       d.vocab_size, start, self.device)
            else:
                dec_ids = prepare_decoder_input_ids(mk["decoder_input_ids"], B, K, d.vocab_size, start, self.device)
        n0 = 1 if dec_ids is None else dec_ids.shape[1]
        # num_return_sequences: the output batch is B * N, take n of description b at row b * N + n.  The encoder ran (and the
        # cross-attention K/V are projected) once per description; what is per row -- a self-attention prompt prefix, the code
        # prefix of a continuation -- is expanded per take.
        if N > 1:
            if prompt_hidden is not None:
                prompt_hidden = prompt_hidden.repeat_interleave(N, dim=0)
                prompt_mask = None if prompt_mask is None else prompt_mask.repeat_interleave(N, dim=0)
            if dec_ids is not None:
                dec_ids = expand_takes(dec_ids, B, K, N)
            if input_lens is not None:
                input_lens = input_lens.repeat_interleave(N)

        # generated length (:3458-3469): max_new_tokens wins over max_length (both count the n0 input columns)
        if gc.max_new_tokens is not None:
            max_length = int(gc.max_new_tokens) + n0
        else:
            max_length = int(user_max_length if user_max_length is not None else gc.max_length)
        if max_length < 2:
            raise ValueError(f"max_length must allow at least one new token, got {max_length}")
        if dec_ids is not None:
            check_continuation_length(n0, P, max_length, d.max_position_embeddings)
        # the caller's processors / criteria are merged with the built-in ones like :3540-3552, on the host-driven loop
        sampling = self._sampling(gc, n0, max_length, seed, suppress_special, row_base, logits_processor, stopping_criteria)
        # output_scores / output_logits exist only in the dict return, as in transformers; without it nothing is recorded
        want_scores = bool(gc.return_dict_in_generate and gc.output_scores)
        want_logits = bool(gc.return_dict_in_generate and gc.output_logits)
        BN = B * N
        outputs = StepOutputs(BN * K, d.vocab_size, self.device, want_scores, want_logits) if (want_scores or want_logits) else None
        probes = StepProbes(d.num_hidden_layers, BN, d.num_attention_heads, S, d.hidden_size, P, n0, self.dtype, self.device, want_attn,
                            want_hidden) if want_attn or want_hidden else None
        align = StepAlignment(align_heads, BN, max_length - n0, text_key0, text_len, self.device) if want_ts else None
        recorders = [r for r in (outputs, align, probes) if r is not None]
        # The fused decode-step kernels hold one 32-row tile: a larger batch runs as consecutive shards of <= 32 rows through the
        # same session, each whole groups of takes (take_shards).  The result is the one the whole batch would give: the Philox
        # draw is keyed by the global row (row_base), the processors' state is per utterance, and a finished utterance emits pad
        # ids until the longest one ends.  The host-driven loop and a streamer run the batch as one session.
        limit = None if sampling.processors or sampling.criteria or streamer is not None else self._fused_batch_limit()
        parts = [self._run_token_loop(enc_hidden, attention_mask, prompt_hidden, prompt_mask, dec_ids, sampling, shard, recorders, streamer,
                                      input_lens)
                 for shard in take_shards(B, N, limit)]
        output_ids = parts[0]
        if len(parts) > 1:
            n = max(t.shape[1] for t in parts)
            output_ids = torch.cat([torch.nn.functional.pad(t, (0, n - t.shape[1]), value=d.pad_token_id) for t in parts], dim=0)
        B = BN   # from here on the batch is the B * N takes

        # apply the stashed delay mask, then keep only the free cells (:3586-3597); both masks come from the whole decoder input,
        # so a continuation's codes begin with its prefix frames
        if input_lens is None:
            mask_src = output_ids[:, :1] if dec_ids is None else dec_ids
            output_ids, codes = self._codes_from_raw(output_ids, mask_src, max_length)
        else:
            output_ids, codes = self._ragged_codes_from_raw(output_ids, dec_ids, input_lens, max_length)
        audio_codes = codes[None, ...]  # frame dim (:3600)

        # The reference decodes sample by sample when any bos/pad/eos id survived (:3615-3619).  Ids in
        # (codebook_size, vocab) other than those (reachable on untrained weights, quirk Q5) would make its
        # embedding lookup fail; here any id >= codebook_size takes the per-sample filtering path.
        cs = self.config.audio_encoder.codebook_size
        decode_sequentially = bool((audio_codes >= cs).any())
        if not decode_sequentially and codes.shape[-1] > 0:
            vals = self.audio_encoder.decode(audio_codes=audio_codes, audio_scales=[None] * B).audio_values.squeeze(1)
            lengths = [vals.shape[1]] * B
            output_values = vals
        else:
            # the reference's per-sample loop (:3620-3647) as one ragged codec call over each row's valid frames
            output_values, lengths = codes_to_waveform(self.audio_encoder, codes, cs, self.dtype)
        if gc.return_dict_in_generate or return_codes:
            out = GenerateOutput(sequences=output_values, audios_length=lengths, audio_codes=codes, raw_ids=output_ids)
            if outputs is not None:   # one entry per generated column: column n0 + t was drawn from entry t
                rec = outputs.result(output_ids.shape[1] - n0)
                out.update(scores=rec.get("scores"), logits=rec.get("logits"))
            if probes is not None:
                out.update(probes.result(output_ids.shape[1] - n0))
                if want_attn:
                    out.update(encoder_attentions=getattr(eo, "attentions", None))
                if want_hidden:
                    out.update(encoder_hidden_states=getattr(eo, "hidden_states", None))
            if want_ts:
                out.update(self._token_timestamps(align, output_ids, n0, text_mask, N))
            if gc.return_dict_in_generate:
                return out
            return output_values, out
        return output_values

    # -- continuous batching -----------------------------------------------------------------------
    @torch.no_grad()
    def generate_continuous(self, input_ids=None, attention_mask=None, prompt_input_ids=None, prompt_attention_mask=None,
                            batch_size: int = 32, refill_every: int = 16, seed=0, return_codes: bool = False, streamer=None,
                            logits_processor=None, stopping_criteria=None, stream: bool = False, **kwargs) -> ContinuousRun:
        """Generate N requests through `batch_size` slots of one live session, refilling a finished request's slot with the next
        request while the others keep decoding.  Returns a ContinuousRun that yields (request index, waveform) as requests finish,
        (request index, waveform, codes [K, T_i]) with return_codes=True.

        The requests come as one generate() call's inputs (padded descriptions or `encoder_outputs`, prompts, masks) and share its
        generation settings; max_length / max_new_tokens count in each request's own columns.  Request i draws with Philox key i
        (substream i * K + k), the key generate() over the whole list gives row i.  Its codes and waveform equal that row's bit
        for bit when generate()'s shards take the prefill kernels a batch_size-row batch takes: always in fp32; in bf16 when every
        shard of generate() (32 rows, and the remainder) and a batch_size-row batch are all at or all below the wgmma GEMM's 128
        rows, for both (P + 1) and S rows per request.  With N = 33 and P < 127, for example, generate() runs the last request in a
        1-row shard below 128 rows, so its bits differ, as they would between generate() calls of different batch sizes.  The text
        encoder runs once over the whole list before the first step, as in generate(): the first audio waits for all N
        descriptions, and the encoder states of all N stay in memory (N x S x H in the model dtype).

        Every `refill_every` decode steps a boundary reads every slot's outcome, computed on the device, in one host sync.  It cuts
        the finished requests' codes out of the history (the delay pattern undone as generate() does), prefills the next requests
        on a second session of batch_size rows (padded with the last request, so one prefill serves the whole refill and its GEMMs
        take a batch_size-row batch's kernels), draws their first column there and imports them into the free slots
        (ptts_session_import_rows).  The batch column is then rebased (rebase_slots, ptts_generate_set_slots), the next interval
        is enqueued, and the finished requests' valid frames go through one ragged codec call behind it (the codec's range check
        waits for that interval, which the next boundary waits for anyway).  Finished rows keep
        decoding PAD until their boundary, so the live session holds max_length + refill_every columns.  Raises ValueError for what
        check_continuous_generate lists.  This is a ContinuousEngine (continuous_engine()) of min(batch_size, N) slots with every
        request submitted up front, stepped until idle.

        stream=True yields each request's audio while it is generated: events (request index, chunk, final), or (request index,
        chunk, final, codes) with return_codes=True, where codes is the [K, T_i] tensor on the final event and None before it.
        Chunks are 1-D device tensors in the model dtype; a request's chunks, in the order yielded, concatenate to the waveform
        stream=False yields for it, bit for bit, and its one final event is its last.  At every boundary each slot's complete
        valid frames so far (slot_outputs(live=True)) give a codec window (stream_windows): the frames whose samples no later
        frame can change are emitted, the rest wait for their right context; a request that ends emits its remainder.  The
        windows of all slots go through one windowed codec call (DACModel._decode_windows), enqueued before the refill and the
        next interval, and the events are yielded in slot order.  A request's first chunk comes at the first boundary that has
        more than dac_dependency_radius (10 for the 44.1 kHz codec) valid frames of it."""
        check_continuous_counts(stream, batch_size, refill_every)
        gc, mk, max_length, suppress_special = continuous_settings(self, kwargs, streamer, logits_processor, stopping_criteria)
        enc_hidden, enc_mask, prompt_hidden, prompt_mask, _, _ = self._conditioning(
            "generate_continuous", input_ids, attention_mask, mk.get("encoder_outputs"), prompt_input_ids, prompt_attention_mask,
            mk.get("prompt_hidden_states"), cross_prompt_after_encoder_outputs=True)
        sampling = self._sampling(gc, 1, max_length, seed, suppress_special)
        N, S = enc_hidden.shape[0], enc_hidden.shape[1]
        P = 0 if prompt_hidden is None else prompt_hidden.shape[1]
        engine = ContinuousEngine(self, sampling, max(1, min(batch_size, N)), refill_every, S, P, stream, bool(return_codes))
        row = lambda t, i: None if t is None else t[i:i + 1]
        for i in range(N):
            engine._submit(enc_hidden[i:i + 1], row(enc_mask, i), row(prompt_hidden, i), row(prompt_mask, i), max_length)
        return ContinuousRun(engine)

    @torch.no_grad()
    def continuous_engine(self, batch_size: int = 32, refill_every: int = 16, max_description_length: Optional[int] = None,
                          max_prompt_length: int = 0, stream: bool = False, return_codes: bool = False, seed=0, streamer=None,
                          logits_processor=None, stopping_criteria=None, **kwargs) -> ContinuousEngine:
        """An online ContinuousEngine: `batch_size` slots of one live session sized for the generation settings' max_length (the
        engine's bound; each request may ask for less), descriptions of up to max_description_length positions (on a
        prompt_cross_attention checkpoint, description and prompt together) and prompts of up to max_prompt_length.  It takes
        generate_continuous()'s settings and refuses what it refuses; the requests' inputs go to submit().  Nothing is decoded
        until step()."""
        check_continuous_counts(stream, batch_size, refill_every)
        for name, v in (("max_description_length", max_description_length), ("max_prompt_length", max_prompt_length)):
            if isinstance(v, bool) or not isinstance(v, int) or v < (1 if name == "max_description_length" else 0):
                raise ValueError(f"{name} must be a {'positive' if name == 'max_description_length' else 'non-negative'} int, got {v!r}")
        gc, mk, max_length, suppress_special = continuous_settings(self, kwargs, streamer, logits_processor, stopping_criteria)
        inputs = sorted(k for k in ("input_ids", "attention_mask", "prompt_input_ids", "prompt_attention_mask", "prompt_hidden_states",
                                    "encoder_outputs", "padding_mask") if mk.get(k) is not None)
        if inputs:
            raise ValueError(f"continuous_engine() takes generation settings; the requests' inputs ({', '.join(inputs)}) go to submit()")
        sampling = self._sampling(gc, 1, max_length, seed, suppress_special)
        return ContinuousEngine(self, sampling, batch_size, refill_every, max_description_length, max_prompt_length, stream,
                                bool(return_codes))
