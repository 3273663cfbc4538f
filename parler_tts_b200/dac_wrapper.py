"""DACModel: the reference's codec wrapper surface, backed by the sm_90a DAC kernels.

Mirrors parler_tts/dac_wrapper/modeling_dac.py:14-164:
  DACModel.encode(input_values, padding_mask=None, bandwidth=None, return_dict=None, n_quantizers=None, sample_rate=None) (:33-104)
  DACModel.decode(audio_codes, audio_scales, padding_mask=None, return_dict=None)   (:106-142), plus frame_lengths= for ragged
  batches (one codec call for utterances of different lengths)
Weights: either folded tensors under transformers-DacModel style keys (decoder.conv1.weight, encoder.block.0.res_unit1..., ...)
or descript-audio-codec checkpoint keys with weight-norm parameters (weight_g / weight_v, or
parametrizations.weight.original0/1), folded here as w = g * v / ||v|| (reference :148-157).  The encoder's weights go to a
blob of their own; a state dict without them (decode only) stays valid, and encode then raises.
"""
from __future__ import annotations
import ctypes as C
import math
import numbers
import re
from dataclasses import dataclass

import torch

from . import _lib
from .configuration import DACConfig


@dataclass
class DACDecoderOutput:
    """Stands in for transformers' EncodecDecoderOutput (audio_values [B, 1, samples])."""
    audio_values: torch.Tensor = None

    def __getitem__(self, i):
        return (self.audio_values,)[i]


@dataclass
class DACEncoderOutput:
    """Stands in for transformers' EncodecEncoderOutput (audio_codes [1, B, K, T], audio_scales [None])."""
    audio_codes: torch.Tensor = None
    audio_scales: list = None

    def __getitem__(self, i):
        return (self.audio_codes, self.audio_scales)[i]


def _dac_tensor_list(cfg: DACConfig) -> list[str]:
    """(id -> key) table in the order csrc/dac.h::make_dac_layout enumerates tensors."""
    names = []
    for i in range(cfg.num_codebooks):
        q = f"quantizer.quantizers.{i}."
        names += [q + "codebook.weight", q + "out_proj.weight", q + "out_proj.bias"]
    names += ["decoder.conv1.weight", "decoder.conv1.bias"]
    for bi in range(len(cfg.decoder_rates)):
        p = f"decoder.block.{bi}."
        names += [p + "snake1.alpha", p + "conv_t1.weight", p + "conv_t1.bias"]
        for r in (1, 2, 3):
            u = p + f"res_unit{r}."
            names += [u + "snake1.alpha", u + "conv1.weight", u + "conv1.bias", u + "snake2.alpha", u + "conv2.weight", u + "conv2.bias"]
    names += ["decoder.snake1.alpha", "decoder.conv2.weight", "decoder.conv2.bias"]
    return names


def _fold_weight_norm(sd: dict[str, torch.Tensor]) -> dict[str, torch.Tensor]:
    """g * v / ||v|| over all dims but 0 (torch weight_norm default dim=0), in fp32."""
    out = {}
    pairs = {}
    for k, v in sd.items():
        m = re.match(r"(.*)\.(weight_g|weight_v|parametrizations\.weight\.original0|parametrizations\.weight\.original1)$", k)
        if m:
            kind = "g" if (m.group(2).endswith("_g") or m.group(2).endswith("original0")) else "v"
            pairs.setdefault(m.group(1), {})[kind] = v
        else:
            out[k] = v
    for base, gv in pairs.items():
        g, v = gv["g"].float(), gv["v"].float()
        norm = v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))
        out[base + ".weight"] = g * v / norm
    return out


def _from_descript_keys(sd: dict[str, torch.Tensor], n_blocks: int) -> dict[str, torch.Tensor]:
    """descript-audio-codec module paths -> the transformers-DacModel style keys used internally.

    descript layout: decoder.model = [WNConv1d, DecoderBlock x n, Snake1d, WNConv1d, Tanh];
    DecoderBlock.block = [Snake1d, WNConvTranspose1d, ResidualUnit x 3]; ResidualUnit.block =
    [Snake1d, WNConv1d(k7), Snake1d, WNConv1d(k1)]."""
    out = {}
    for k, v in sd.items():
        if k.startswith("quantizer."):
            out[k] = v
            continue
        m = re.match(r"decoder\.model\.(\d+)\.(.*)$", k)
        if not m:
            continue
        i, rest = int(m.group(1)), m.group(2)
        if i == 0:
            out["decoder.conv1." + rest] = v
        elif 1 <= i <= n_blocks:
            bi = i - 1
            mm = re.match(r"block\.(\d+)\.(.*)$", rest)
            j, r2 = int(mm.group(1)), mm.group(2)
            p = f"decoder.block.{bi}."
            if j == 0:
                out[p + "snake1." + r2] = v
            elif j == 1:
                out[p + "conv_t1." + r2] = v
            else:
                m3 = re.match(r"block\.(\d+)\.(.*)$", r2)
                u, r3 = int(m3.group(1)), m3.group(2)
                name = {0: "snake1.", 1: "conv1.", 2: "snake2.", 3: "conv2."}[u]
                out[p + f"res_unit{j - 1}." + name + r3] = v
        elif i == n_blocks + 1:
            out["decoder.snake1." + rest] = v
        elif i == n_blocks + 2:
            out["decoder.conv2." + rest] = v
    return out


def _dac_encoder_tensor_list(cfg: DACConfig) -> list[str]:
    """(id -> key) table of the encoder blob, in the order csrc/dac.h::make_dac_enc_layout enumerates tensors."""
    names = ["encoder.conv1.weight", "encoder.conv1.bias"]
    for bi in range(len(cfg.encoder_rates)):
        p = f"encoder.block.{bi}."
        for r in (1, 2, 3):
            u = p + f"res_unit{r}."
            names += [u + "snake1.alpha", u + "conv1.weight", u + "conv1.bias", u + "snake2.alpha", u + "conv2.weight", u + "conv2.bias"]
        names += [p + "snake1.alpha", p + "conv1.weight", p + "conv1.bias"]
    names += ["encoder.snake1.alpha", "encoder.conv2.weight", "encoder.conv2.bias"]
    for i in range(cfg.num_codebooks):
        q = f"quantizer.quantizers.{i}."
        names += [q + "in_proj.weight", q + "in_proj.bias", q + "codebook.weight"]
    return names


# descript's Encoder is one Sequential (encoder.block.N.weight, encoder.block.N.block.M...); transformers' DacEncoder names its
# modules (encoder.block.N.res_unitM..., encoder.conv1...)
_DESCRIPT_ENCODER_KEY = re.compile(r"encoder\.block\.\d+\.(block\.|weight$|bias$|alpha$)")


def _from_descript_encoder_keys(sd: dict[str, torch.Tensor], n_blocks: int) -> dict[str, torch.Tensor]:
    """descript-audio-codec encoder paths -> the transformers-DacModel style keys used internally.

    descript layout: encoder.block = [WNConv1d(k7), EncoderBlock x n, Snake1d, WNConv1d(k3)]; EncoderBlock.block =
    [ResidualUnit x 3, Snake1d, WNConv1d(k=2s, stride s)]; ResidualUnit.block = [Snake1d, WNConv1d(k7), Snake1d, WNConv1d(k1)]."""
    out = {}
    for k, v in sd.items():
        m = re.match(r"encoder\.block\.(\d+)\.(.*)$", k)
        if not m:
            continue
        i, rest = int(m.group(1)), m.group(2)
        if i == 0:
            out["encoder.conv1." + rest] = v
        elif 1 <= i <= n_blocks:
            mm = re.match(r"block\.(\d+)\.(.*)$", rest)
            if not mm:
                continue
            j, r2 = int(mm.group(1)), mm.group(2)
            p = f"encoder.block.{i - 1}."
            if j < 3:
                m3 = re.match(r"block\.(\d+)\.(.*)$", r2)
                u, r3 = int(m3.group(1)), m3.group(2)
                name = {0: "snake1.", 1: "conv1.", 2: "snake2.", 3: "conv2."}[u]
                out[p + f"res_unit{j + 1}." + name + r3] = v
            elif j == 3:
                out[p + "snake1." + r2] = v
            elif j == 4:
                out[p + "conv1." + r2] = v
        elif i == n_blocks + 1:
            out["encoder.snake1." + rest] = v
        elif i == n_blocks + 2:
            out["encoder.conv2." + rest] = v
    return out


def _encoder_state_dict(sd: dict[str, torch.Tensor], n_blocks: int) -> dict[str, torch.Tensor]:
    """The encoder and quantizer keys of a folded state dict, in transformers-DacModel style whichever layout it came in."""
    if any(_DESCRIPT_ENCODER_KEY.match(k) for k in sd):
        out = _from_descript_encoder_keys(sd, n_blocks)
    else:
        out = {k: v for k, v in sd.items() if k.startswith("encoder.")}
    out.update({k: v for k, v in sd.items() if k.startswith("quantizer.")})
    return out


def _row_lengths(lengths, B: int, lo: int, hi: int, name: str) -> torch.Tensor:
    """Per-row lengths (ints or an integer tensor) -> int32 [B] on the host; ValueError for a wrong shape, dtype or a value
    outside [lo, hi]."""
    if isinstance(lengths, torch.Tensor):
        if lengths.is_floating_point() or lengths.is_complex() or lengths.dtype == torch.bool:
            raise ValueError(f"{name} must hold integers, got {lengths.dtype}")
        n = lengths.detach().cpu()
    else:
        vals = list(lengths)
        if not all(isinstance(v, numbers.Integral) and not isinstance(v, bool) for v in vals):
            raise ValueError(f"{name} must hold integers, got {vals}")
        n = torch.tensor([int(v) for v in vals], dtype=torch.int64)
    if n.shape != (B,):
        raise ValueError(f"{name} must have shape [{B}] (one length per batch row), got {tuple(n.shape)}")
    if bool(((n < lo) | (n > hi)).any()):
        raise ValueError(f"{name} must lie in [{lo}, {hi}], got {n.tolist()}")
    return n.to(torch.int32)


def _frame_lengths(frame_lengths, B: int, T: int) -> torch.Tensor:
    """DACModel.decode's frame_lengths -> int32 [B] on the host; ValueError for a wrong shape, dtype or value outside [0, T]."""
    return _row_lengths(frame_lengths, B, 0, T, "frame_lengths")


def _sample_lengths(sample_lengths, B: int, samples: int) -> torch.Tensor:
    """DACModel.encode's sample_lengths -> int32 [B] on the host; ValueError for a wrong shape, dtype or value outside
    [1, samples]."""
    return _row_lengths(sample_lengths, B, 1, samples, "sample_lengths")


class DACModel:
    config_class = DACConfig
    main_input_name = "input_values"

    def __init__(self, config: DACConfig, device="cuda", dtype=torch.float32):
        self.config = config
        self.device = torch.device(device)
        self.dtype = dtype
        self._c = _lib.DacConfigC()
        self._c.n_codebooks = config.num_codebooks
        self._c.codebook_size = config.codebook_size
        self._c.codebook_dim = config.codebook_dim
        self._c.latent_dim = config.latent_dim
        self._c.decoder_dim = config.decoder_dim
        self._c.n_blocks = len(config.decoder_rates)
        for i, s in enumerate(config.decoder_rates):
            self._c.strides[i] = int(s)
        self._c.dtype = _lib.dtype_code(dtype)
        self.hop_length = math.prod(config.decoder_rates)
        # the packed weight blob exists from construction on (zeros until load_state_dict / a broadcast fills it), so that
        # every rank of a sharded run owns a buffer of the right size for the init broadcast (dist.broadcast_model_weights)
        nbytes = C.c_int64()
        _lib.check(_lib.lib().ptts_dac_blob_bytes(C.byref(self._c), C.byref(nbytes)))
        self.blob = torch.zeros(nbytes.value, dtype=torch.uint8, device=self.device)
        self.loaded = False
        self._ws = None
        # the encoder blob, likewise from construction on; None when the config has no usable encoder (encoder_dim = 0, or
        # rates the kernels do not take, such as a hop that differs from the decoder's): decode still works, encode raises
        self.encoder_blob = None
        self.encoder_loaded = False
        self._encoder_error = "the config has no encoder (encoder_dim = 0)"
        self._enc_ws = None
        rates = list(getattr(config, "encoder_rates", None) or [])
        if getattr(config, "encoder_dim", 0) and len(rates) > 8:
            self._encoder_error = f"{len(rates)} encoder blocks (at most 8)"
        elif getattr(config, "encoder_dim", 0):
            self._c.encoder_dim = int(config.encoder_dim)
            self._c.n_enc_blocks = len(rates)
            for i, s in enumerate(rates):
                self._c.encoder_rates[i] = int(s)
            try:
                _lib.check(_lib.lib().ptts_dac_encoder_blob_bytes(C.byref(self._c), C.byref(nbytes)))
                self.encoder_blob = torch.zeros(nbytes.value, dtype=torch.uint8, device=self.device)
                self._encoder_error = None
            except ValueError as e:
                self._encoder_error = str(e)

    # -- weights -----------------------------------------------------------------------------------
    def load_state_dict(self, sd: dict[str, torch.Tensor], strict: bool = True):
        sd = {(k[len("model."):] if k.startswith("model.") else k): v for k, v in sd.items()}
        sd = _fold_weight_norm(sd)
        enc_sd = _encoder_state_dict(sd, len(getattr(self.config, "encoder_rates", None) or []))
        if any(k.startswith("decoder.model.") for k in sd):
            sd = _from_descript_keys(sd, len(self.config.decoder_rates))
        names = _dac_tensor_list(self.config)
        missing = [n for n in names if n not in sd]
        if missing and strict:
            raise ValueError(f"DACModel.load_state_dict: missing keys {missing[:5]}{'...' if len(missing) > 5 else ''}")
        lib = _lib.lib()
        n = C.c_int32()
        _lib.check(lib.ptts_dac_num_tensors(C.byref(self._c), C.byref(n)))
        assert n.value == len(names), (n.value, len(names))
        self.blob.zero_()
        for i, name in enumerate(names):
            if name not in sd:
                continue
            t = sd[name].to(device=self.device)
            if t.dtype not in (torch.float32, torch.bfloat16):
                t = t.float()
            t = t.contiguous()
            _lib.check(lib.ptts_dac_pack(C.byref(self._c), _lib.ptr(self.blob), i, _lib.ptr(t), _lib.dtype_code(t.dtype),
                                         t.numel(), _lib.stream_ptr()))
        torch.cuda.current_stream().synchronize()  # staging tensors above go out of scope
        self.loaded = True
        self._load_encoder(enc_sd, strict)
        return self

    def _load_encoder(self, sd: dict[str, torch.Tensor], strict: bool):
        """Pack the encoder keys of `sd` (from _encoder_state_dict) into the encoder blob; none present: decode only."""
        self.encoder_loaded = False
        if self.encoder_blob is None or not any(k.startswith("encoder.") for k in sd):
            return
        names = _dac_encoder_tensor_list(self.config)
        missing = [n for n in names if n not in sd]
        if missing and strict:
            raise ValueError(f"DACModel.load_state_dict: missing encoder keys {missing[:5]}{'...' if len(missing) > 5 else ''}")
        lib = _lib.lib()
        n = C.c_int32()
        _lib.check(lib.ptts_dac_encoder_num_tensors(C.byref(self._c), C.byref(n)))
        assert n.value == len(names), (n.value, len(names))
        self.encoder_blob.zero_()
        for i, name in enumerate(names):
            if name not in sd:
                continue
            t = sd[name].to(device=self.device)
            if t.dtype not in (torch.float32, torch.bfloat16):
                t = t.float()
            t = t.contiguous()
            _lib.check(lib.ptts_dac_encoder_pack(C.byref(self._c), _lib.ptr(self.encoder_blob), i, _lib.ptr(t), _lib.dtype_code(t.dtype),
                                                 t.numel(), _lib.stream_ptr()))
        torch.cuda.current_stream().synchronize()
        self.encoder_loaded = True

    def to(self, *args, **kwargs):
        return self

    def eval(self):
        return self

    # -- reference surface -------------------------------------------------------------------------
    @torch.no_grad()
    def encode(self, input_values, padding_mask=None, bandwidth=None, return_dict=None, n_quantizers=None, sample_rate=None,
               sample_lengths=None):
        """input_values [B, 1, samples] -> DACEncoderOutput(audio_codes [1, B, n_q, ceil(samples / hop)] int64, audio_scales [None]).

        One chunk, right zero-padded to the hop like model.preprocess (:64); n_q = n_quantizers or every codebook.
        `padding_mask` and `bandwidth` are unused, as in the reference.  Float32 or model-dtype audio; it is rounded to the
        model dtype before the first conv.

        sample_lengths (ints or an integer tensor of shape [B], each in [1, samples]) encodes a ragged batch in one call: row b
        equals the encode of input_values[b:b+1, :, :sample_lengths[b]] alone, bit for bit, in its first
        F_b = ceil(sample_lengths[b] / hop) frames, and holds codebook_size (no frame) after them.  Samples past a row's length
        are never read and may hold anything."""
        if not isinstance(input_values, torch.Tensor) or input_values.dim() != 3:
            raise ValueError(f"input_values must be [batch, channels, samples], got {getattr(input_values, 'shape', type(input_values))}")
        B, channels, n = input_values.shape
        if channels < 1 or channels > 2:
            raise ValueError(f"Number of audio channels must be 1 or 2, but got {channels}")
        if channels == 2:
            raise ValueError("the DAC encoder takes mono audio [B, 1, samples] (its first conv has one input channel), got 2 channels")
        if sample_rate is not None and int(sample_rate) != self.config.sampling_rate:
            raise ValueError(f"sample_rate {sample_rate} differs from the codec's {self.config.sampling_rate}")
        if B == 0 or n == 0:
            raise ValueError(f"input_values is empty: shape {tuple(input_values.shape)}")
        if not input_values.is_floating_point():
            raise ValueError(f"input_values must be a floating-point waveform, got {input_values.dtype}")
        K = self.config.num_codebooks
        n_q = K if n_quantizers is None else int(n_quantizers)
        if not 1 <= n_q <= K:
            raise ValueError(f"n_quantizers must lie in 1..{K}, got {n_quantizers}")
        lengths = None if sample_lengths is None else _sample_lengths(sample_lengths, B, n)
        codes, _ = self._encode(input_values[:, 0, :], n_q, sample_lengths=lengths)
        codes = codes[None]
        if return_dict is False:
            return (codes, [None])
        return DACEncoderOutput(codes, [None])

    def _encode(self, audio: torch.Tensor, n_q: int, return_latents: bool = False, sample_lengths=None):
        """audio [B, samples] -> (codes [B, n_q, T] int64, encoder output [B, T, latent_dim] in the model dtype or None).
        sample_lengths: None, or an integer tensor [B] already checked to lie in [1, samples] (encode's ragged batch; the
        latents past a row's frames are 0)."""
        if self.encoder_blob is None:
            raise ValueError(f"DACModel.encode is not available for this config: {self._encoder_error}")
        if not (self.encoder_loaded and self.loaded):
            raise RuntimeError("DACModel has no encoder weights loaded (a decode-only state dict): encode needs the encoder.* and "
                               "quantizer.quantizers.N.{in_proj,codebook,out_proj} weights")
        audio = audio.to(device=self.device, dtype=self.dtype).contiguous()
        B, n = audio.shape
        T = -(-n // self.hop_length)
        lib = _lib.lib()
        need = C.c_int64()
        _lib.check(lib.ptts_dac_encode_workspace_bytes(C.byref(self._c), B, n, C.byref(need)))
        if self._enc_ws is None or self._enc_ws.numel() < need.value:
            self._enc_ws = torch.empty(need.value, dtype=torch.uint8, device=self.device)
        codes = torch.empty(B, n_q, T, dtype=torch.int64, device=self.device)
        latents = torch.empty(B, T, self.config.latent_dim, dtype=self.dtype, device=self.device) if return_latents else None
        lengths = None if sample_lengths is None else sample_lengths.to(device=self.device, dtype=torch.int32).contiguous()
        _lib.check(lib.ptts_dac_encode2(C.byref(self._c), _lib.ptr(self.blob), _lib.ptr(self.encoder_blob), _lib.ptr(self._enc_ws),
                                        self._enc_ws.numel(), _lib.ptr(audio), B, n, _lib.ptr(lengths), n_q, _lib.ptr(codes),
                                        _lib.ptr(latents), _lib.stream_ptr()))
        return codes, latents

    @torch.no_grad()
    def decode(self, audio_codes, audio_scales=None, padding_mask=None, return_dict=None, frame_lengths=None):
        """audio_codes [1, B, K, T] int64 (CUDA) -> DACDecoderOutput(audio_values [B, 1, hop*T]).

        frame_lengths (ints or an integer tensor of shape [B], each in [0, T]) decodes a ragged batch in one call: row b equals
        the decode of audio_codes[:, b:b+1, :, :frame_lengths[b]] alone, bit for bit, in samples [0, hop*frame_lengths[b]) and is
        0 after them.  Codes at frames >= frame_lengths[b] are never read and may hold anything (EOS / pad ids included).
        `padding_mask` is accepted and unused, as in the reference."""
        if not self.loaded:
            raise RuntimeError("DACModel has no weights loaded")
        if len(audio_codes) != 1:
            raise ValueError(f"Expected one frame, got {len(audio_codes)}")
        codes = audio_codes.squeeze(0)
        if codes.dim() != 3 or codes.shape[1] != self.config.num_codebooks:
            raise ValueError(f"audio_codes must be [1, B, {self.config.num_codebooks}, T], got {tuple(audio_codes.shape)}")
        codes = codes.to(device=self.device, dtype=torch.int64).contiguous()
        B, K, T = codes.shape
        if T == 0 or B == 0:
            raise ValueError("audio_codes is empty")
        lengths = None if frame_lengths is None else _frame_lengths(frame_lengths, B, T)
        bad = (codes < 0) | (codes >= self.config.codebook_size)
        if lengths is not None:
            lengths = lengths.to(self.device)
            bad &= torch.arange(T, device=self.device) < lengths[:, None, None]   # only frames inside each row are read
        if bool(bad.any()):
            raise IndexError("audio code out of range for the codebook (the reference's embedding lookup raises too)")
        lib = _lib.lib()
        need = C.c_int64()
        _lib.check(lib.ptts_dac_workspace_bytes(C.byref(self._c), B, T, C.byref(need)))
        if self._ws is None or self._ws.numel() < need.value:
            self._ws = torch.empty(need.value, dtype=torch.uint8, device=self.device)
        audio = torch.empty(B, 1, T * self.hop_length, dtype=self.dtype, device=self.device)
        _lib.check(lib.ptts_dac_decode2(C.byref(self._c), _lib.ptr(self.blob), _lib.ptr(self._ws), self._ws.numel(),
                                        _lib.ptr(codes), B, T, _lib.ptr(lengths), _lib.ptr(audio), _lib.stream_ptr()))
        if return_dict is False:
            return (audio,)
        return DACDecoderOutput(audio)

    def _decode_windows(self, codes: torch.Tensor, windows: list) -> torch.Tensor:
        """Streamed decode of one window per row: codes [B, K, T_codes] int64 (CUDA, contiguous), windows [(start, n, lo, hi)] * B.
        Row b's samples of window frames [lo, hi) equal, bit for bit, those of decode() on codes[b, :, start:start + n] alone;
        the rest of the row is 0.  Returns a fresh [B, hop * max n] tensor.  Each layer computes only the rows those samples
        depend on (ptts_dac_decode3).  No range check (it would wait for the device): the ids inside the windows must be
        codebook ids."""
        B, _, T_codes = codes.shape
        T = max(w[1] for w in windows)
        lib = _lib.lib()
        need = C.c_int64()
        _lib.check(lib.ptts_dac_workspace_bytes(C.byref(self._c), B, T, C.byref(need)))
        if self._ws is None or self._ws.numel() < need.value:
            self._ws = torch.empty(need.value, dtype=torch.uint8, device=self.device)
        ranges = torch.tensor(windows, dtype=torch.int32).t().contiguous().pin_memory().to(self.device, non_blocking=True)   # [4, B]
        audio = torch.empty(B, T * self.hop_length, dtype=self.dtype, device=self.device)
        _lib.check(lib.ptts_dac_decode3(C.byref(self._c), _lib.ptr(self.blob), _lib.ptr(self._ws), self._ws.numel(), _lib.ptr(codes), B,
                                        T_codes, T, _lib.ptr(ranges[0]), _lib.ptr(ranges[1]), _lib.ptr(ranges[2]), _lib.ptr(ranges[3]),
                                        _lib.ptr(audio), _lib.stream_ptr()))
        return audio

    def forward(self, tensor):
        raise ValueError("`DACModel.forward` not implemented yet")
