"""Multi-GPU: one process per GPU, the generation batch sharded by utterance (SURVEY.md 8e).

The path has no per-step exchange -- utterances are independent -- so the only collective is one
broadcast of the packed weight blobs from rank 0 at init (NCCL over NVLink on GPUs; the same code runs
on gloo/CPU tensors in the world_size-2 unit tests).  Sampling uses per-row Philox substreams keyed by
the GLOBAL row index (ptts_gen_params.row_base = first local utterance x num_codebooks; generate(row_base=...)
or shard_row_base() below), so the draws of an utterance do not depend on the number of shards.
"""
from __future__ import annotations
import torch
import torch.distributed as dist


def shard_range(n: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous, balanced rows [lo, hi) of rank; the first n % world ranks take one extra row."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_row_base(n: int, rank: int, world: int, num_codebooks: int) -> int:
    """Global (utterance, codebook) row index of this rank's first row: the `row_base` to pass to generate().  row_base counts
    takes: with generate(num_return_sequences=N) pass shard_row_base(...) * N, so that take j of description b draws the
    substreams of global row (b * N + j) * num_codebooks + k whatever the number of ranks."""
    return shard_range(n, rank, world)[0] * num_codebooks


def shard_batch(tensors: dict, rank: int, world: int) -> dict:
    """Slice every [B, ...] tensor of a generate() kwarg dict to this rank's utterances.  `decoder_input_ids` ([B * K, N] audio
    codes) is split by its K-row groups, one group per utterance, and a list of `input_values` clips by its items."""
    B = next(v.shape[0] for k, v in tensors.items() if isinstance(v, torch.Tensor) and k != "decoder_input_ids")
    lo, hi = shard_range(B, rank, world)
    out = {}
    for k, v in tensors.items():
        if k == "decoder_input_ids" and isinstance(v, torch.Tensor):
            if v.shape[0] % B != 0:
                raise ValueError(f"decoder_input_ids has {v.shape[0]} rows, not a multiple of the batch size {B}")
            K = v.shape[0] // B
            out[k] = v[lo * K:hi * K]
        elif k == "input_values" and isinstance(v, (list, tuple)):   # one clip per utterance (a ragged continuation)
            out[k] = list(v[lo:hi])
        else:
            out[k] = v[lo:hi] if isinstance(v, torch.Tensor) and v.shape[0] == B else v
    return out


def broadcast_blob(blob: torch.Tensor, src: int = 0, group=None) -> torch.Tensor:
    """One collective at init: ship the packed (already repacked) weight bytes from `src` to every rank."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.broadcast(blob, src=src, group=group)
    return blob


def model_weight_tensors(model) -> list[torch.Tensor]:
    """Every device tensor that holds weights, in a fixed order that depends on the CONFIG only (never on what a rank has
    loaded): the packed decoder blob, the packed DAC blob, the prompt embedding table, when the text encoder's width
    differs from the decoder's, enc_to_dec_proj (modeling_parler_tts.py:2388-2392), with config.prompt_cross_attention the
    prompt's position table (:2397-2402), and the DAC encoder blob when the codec config has an encoder.  All exist from
    construction on."""
    ts = [model.decoder.engine.blob, model.audio_encoder.blob, model.embed_prompts_weight]
    if model.enc_to_dec_proj is not None:
        ts += list(model.enc_to_dec_proj)
    if getattr(model, "embed_positions_weight", None) is not None:
        ts.append(model.embed_positions_weight)
    enc_blob = getattr(model.audio_encoder, "encoder_blob", None)
    if enc_blob is not None:
        ts.append(enc_blob)
    return ts


def broadcast_model_weights(model, src: int = 0, group=None):
    """Rank `src` has loaded/packed the checkpoint; the others only constructed the model (zero-filled buffers of the same
    sizes).  Every rank issues the same sequence of broadcasts: one per tensor of model_weight_tensors() plus one flag word."""
    ts = model_weight_tensors(model)
    for t in ts:
        broadcast_blob(t, src, group)
    flags = torch.tensor([int(model.audio_encoder.loaded), int(model._side_loaded), int(getattr(model.audio_encoder, "encoder_loaded", False))],
                         dtype=torch.int32, device=ts[0].device)
    broadcast_blob(flags, src, group)
    loaded = flags.cpu().tolist()
    model.audio_encoder.loaded = bool(loaded[0])
    model._side_loaded = bool(loaded[1])
    if hasattr(model.audio_encoder, "encoder_loaded"):
        model.audio_encoder.encoder_loaded = bool(loaded[2])
    return model


def gather_ragged_audio(audio: torch.Tensor, lengths: list[int], group=None):
    """Host-side concatenation of per-rank ragged outputs -> (list of [n_i] tensors in global batch order)."""
    local = [audio[i, : lengths[i]].cpu() for i in range(audio.shape[0])]
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local
    out = [None] * dist.get_world_size(group)
    dist.all_gather_object(out, local, group=group)
    return [a for part in out for a in part]
