"""The codec's convolutions one launch at a time, against a float64 reference, through the ptts_op_dac_conv hook.

Kernels: 0 is conv_kernel of dac.cu (64 x 64 output tiles, 16-channel K chunks, one serial fmaf chain per output, snake on the
input, bias, residual and tanh fused; bf16 and f32).  1 is conv_tc_kernel of dac_tc.cu (128-row tiles, N tiles of 128 / 96 /
64 / 32 columns, a 3-stage TMA ring of 64-channel K chunks over (tap, chunk) pairs, bias + residual + snake_{alpha_next} in the
epilogue, the ragged zero band written by the producer warp).  2 is final_conv_tanh_kernel (C -> 1, k 7, one thread per
sample).  3 is enc_input_conv_kernel (1 -> C, k 7, raw and snake for the next layer).  The geometry of each launch is built by
dac.h's conv_same / conv_up / conv_super_rows and the weights go through the blob's packs, so both are under test too.

The reference is the layer in float64 with torch's own F.conv1d / F.conv_transpose1d on the values the kernel sees (bf16 or
f32 inputs, weights rounded to the model dtype): conv_same is padding (k-1)/2 dil, the transposed conv stride s padding
ceil(s/2), the strided conv stride s padding s/2.  Nothing in it comes from the kernels' phase, tap or super-row mapping.  The
epilogue rounds where torch's bf16 ops round in the reference module: raw = rn(conv + bias), rn(res + raw),
snake(x) = rn(x + rn(rn(1/rn(alpha + 1e-9)) rn(rn(sin(rn(alpha x)))^2))), final conv rn(tanh(rn(conv + bias))).  rn is one
rounding to bf16 (through fp32: exact for every value rounded that way here -- products of two bf16 fit fp32, and a sum of two
bf16 cannot land on a bf16 midpoint after its fp32 rounding, so the two roundings agree with one).

Bars (u = 2^-24, one fp32 rounding):
  E_acc  = u (n + 32) mass + u |conv + bias|: mass = sum |x||w| (the fp64 conv of |x| with |w|); n chained fp32 additions
           err by at most n u mass whatever their order, products of bf16 are exact in fp32.  n = taps ceil(Cin/16) on the
           wgmma kernel (one fp32 rounding per m64nNk16 step, as test_linear_reference models the MMA paths), taps Cin on the
           serial fmaf chains of kernels 0, 2 and 3; 32 covers the rest, and the last term is the rounding of the bias add.
  bf16:    the kernel's value must be a member of a candidate set.  raw is any bf16 value in [rn(z - E_acc), rn(z + E_acc)]
           (z = conv + bias in fp64) -- one value unless a rounding midpoint lies within reach.  Each raw candidate goes through
           the deterministic bf16 ops (residual add, alpha x, the squares, the product, the add) exactly; sin and tanh may take
           either neighbour only where the fp64 value lies within E_f of a bf16 midpoint, E_f = 2 fp32 ulps of the result +
           2^-22: the accuracy of CUDA's sinf / tanhf (2 ulp) with an absolute floor.  E_f is a property of the contract
           (torch rounds the correctly rounded value): it is not widened to excuse an approximate sine.  On the generic kernel
           an input whose snake is itself ambiguous adds (its candidates' spread) |w| to its outputs' E_acc.
  f32 (kernel 0 only):  |got - ref| <= E_acc + sum |w| delta + 4 u (|ref| + |res|) (+ 2 fp32 ulps of tanhf), delta the input
           snake's error: 2 ulps of sinf (4u relative on sin, 8u on sin^2), the roundings of alpha x (|sin 2ax| |ax| u / alpha),
           of alpha + 1e-9 and 1/. (2u), of s*s and inv*. (2u), and of the final add (u |snake|): 12 u t + the two other terms.

Every output buffer starts as NaN with NaN rows past B * Tout: every element inside the shape must be written (so conv_up's
phases cover [0, T s) exactly once) and everything past it must stay NaN.  Ragged rows (frame_lengths with 0, 1, frames - 1 and
frames) must equal the reference of the row zero-padded past its end, and be exactly 0 past it: on every row for kernels 0 and
2, over the zero band of more than 128 rows for the wgmma kernel (which leaves later tiles unwritten).  The host tests check
that each modelled kernel bug moves its case's reference past the bar on some element (by more than 4x an f32 bar; two or more
bf16 values outside a candidate set, which a member check with one extra neighbour would still catch), and the reference itself
against torch's fp32 conv and against the bf16 oracle's layers.
"""
from __future__ import annotations

import dataclasses
import math

import pytest
import torch
import torch.nn.functional as F

U = 2.0 ** -24
DEV = "cuda"
STATS: dict = {}      # (kernel, dtype) -> [cases, elements, two raw candidates, two sin candidates, worst f32 error / bar]
SWEEP: dict = {}      # kernel -> [largest |alpha x| checked, elements with two sin candidates]


# ---- bf16 helpers ----------------------------------------------------------------------------------------------------------
def rn(t: torch.Tensor) -> torch.Tensor:
    return t.float().bfloat16().double()


def ulp_f32(t: torch.Tensor) -> torch.Tensor:
    e = torch.floor(torch.log2(t.abs().clamp(min=2.0 ** -126)))
    return torch.exp2(e - 23)


def bf_ord(t: torch.Tensor) -> torch.Tensor:
    """bf16 values (float64) -> integers in the same order, adjacent values one apart (+0 and -0 both 0)."""
    b = t.float().bfloat16().view(torch.int16).to(torch.int32)
    return torch.where(b < 0, -(b & 0x7FFF), b)


def bf_from_ord(o: torch.Tensor) -> torch.Tensor:
    b = torch.where(o < 0, (-o) - 32768, o).to(torch.int16)
    return b.view(torch.bfloat16).double()


def inv_of(alpha: torch.Tensor) -> torch.Tensor:
    """rn(1 / rn(alpha + 1e-9)) the way torch's bf16 ops (and the kernels) compute it: fp32 ops, bf16 results."""
    a = alpha.float()
    return (1.0 / (a + 1e-9).bfloat16().float()).bfloat16().double()


def snake_set(r: torch.Tensor, alpha: torch.Tensor, inv: torch.Tensor):
    """bf16 snake of bf16 values r (alpha, inv broadcast over r's last dim): (nearest, lo, hi, sin ambiguous, |alpha x|)."""
    ax = rn(alpha * r)
    s64 = torch.sin(ax)
    ef = 2 * ulp_f32(s64) + 2.0 ** -22
    sn, sn_lo, sn_hi = rn(s64), rn(s64 - ef), rn(s64 + ef)
    a_min = torch.where((sn_lo <= 0) & (sn_hi >= 0), torch.zeros_like(sn), torch.minimum(sn_lo.abs(), sn_hi.abs()))
    a_max = torch.maximum(sn_lo.abs(), sn_hi.abs())

    def fin(a):
        return rn(r + rn(inv * rn(a * a)))
    lo, hi = fin(a_min), fin(a_max)
    return fin(sn.abs()), torch.minimum(lo, hi), torch.maximum(lo, hi), sn_lo != sn_hi, ax.abs()


def tanh_set(r_lo: torch.Tensor, r_hi: torch.Tensor):
    t_lo, t_hi = torch.tanh(r_lo), torch.tanh(r_hi)
    return rn(t_lo - 2 * ulp_f32(t_lo) - 2.0 ** -22), rn(t_hi + 2 * ulp_f32(t_hi) + 2.0 ** -22)


# ---- cases -----------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Case:
    kernel: int                  # 0 conv_kernel, 1 conv_tc_kernel, 2 final conv, 3 input conv
    dtype: torch.dtype
    kind: int                    # 0 conv_same, 1 conv_up, 2 conv_super_rows
    B: int
    Cin: int
    Cout: int
    T: int                       # input rows (kernel 3: output rows)
    taps: int = 7
    d: int = 1                   # dilation (kind 0) or stride
    res: str = "none"            # "none", "sep" or "inplace" (res == out_raw)
    raw: bool = True
    act: bool = False            # kernel 1: snake_{alpha_next} of the output; kernel 0: snake on the input
    tanh: bool = False
    samples: int = 0             # kernel 3 (and kernel 0's encoder input conv): waveform rows
    frames: int = 0              # > 0: ragged, frame_lengths [0, 1, frames - 1, frames, ...]
    alpha: tuple = (0.01, 100.0)
    sweep: bool = False          # |alpha x| over 2^-10 .. 2^12
    sample_rows: bool = False    # compare tile-edge and random rows only
    seed: int = 0

    @property
    def id(self):
        dt = "bf16" if self.dtype == torch.bfloat16 else "f32"
        g = ["same", "up", "super"][self.kind]
        s = f"k{self.kernel}-{dt}-{g}-B{self.B}-{self.Cin}x{self.Cout}-T{self.T}-t{self.taps}d{self.d}"
        for flag, name in ((self.res != "none", "res-" + self.res), (self.act, "act"), (not self.raw, "noraw"),
                           (self.tanh, "tanh"), (self.samples, f"samples{self.samples}"), (self.frames, f"ragged{self.frames}"),
                           (self.sweep, "sweep")):
            if flag:
                s += "-" + name
        return s

    @property
    def tin(self):
        return self.samples if (self.kernel == 3 or self.samples) else self.T

    @property
    def tout(self):
        return self.T * self.d if self.kind == 1 else self.T // self.d if self.kind == 2 else self.T

    @property
    def cin_k(self):             # channels of the kernel's K dimension (super rows: s * C)
        return self.Cin * self.d if self.kind == 2 else self.Cin

    @property
    def n_chain(self):
        taps = 2 if self.kind == 1 else 3 if self.kind == 2 else self.taps
        return taps * math.ceil(self.cin_k / 16) if self.kernel == 1 else taps * self.cin_k

    @property
    def up(self):                # rows per frame at the input and the output
        return self.tin // self.frames, self.tout // self.frames


def bf(kernel, kind, B, Cin, Cout, T, taps=7, d=1, **kw):
    return Case(kernel, torch.bfloat16, kind, B, Cin, Cout, T, taps, d, **kw)


BF, F32 = torch.bfloat16, torch.float32
TC_CASES = [
    # conv_same: every N tile (32 .. 128, multi-tile grids), Cin tails (96, 160) and one K step against the 3-stage ring
    bf(1, 0, 3, 64, 32, 129, 1, 1, act=True),
    bf(1, 0, 1, 96, 64, 127, 7, 1, act=True),
    bf(1, 0, 3, 128, 96, 128, 7, 3, act=True, res="sep"),
    bf(1, 0, 1, 160, 128, 257, 3, 1, act=True),
    bf(1, 0, 3, 160, 160, 129, 7, 9, act=True, res="inplace"),
    bf(1, 0, 3, 96, 320, 1, 7, 1, act=True),
    bf(1, 0, 1, 1536, 1536, 4097, 7, 1, act=True),
    bf(1, 0, 3, 64, 1536, 4097, 1, 1, res="inplace", act=True),
    bf(1, 0, 1, 1536, 32, 257, 7, 9, act=True),
    bf(1, 0, 3, 64, 64, 1, 3, 1, act=True),
    # epilogues: raw only, act only, both; residual separate and in place
    bf(1, 0, 3, 128, 96, 257, 7, 3, raw=True, act=False),
    bf(1, 0, 3, 128, 96, 257, 7, 3, raw=False, act=True),
    bf(1, 0, 3, 128, 96, 257, 7, 3, raw=True, act=True, res="sep"),
    bf(1, 0, 3, 128, 96, 257, 7, 3, raw=True, act=True, res="inplace"),
    bf(1, 0, 1, 96, 160, 129, 1, 1, raw=False, act=True, res="sep"),
    # conv_up: q_count = T + 1 on 127 / 128 / 129
    bf(1, 1, 3, 128, 64, 126, d=2, act=True),
    bf(1, 1, 1, 256, 128, 127, d=4, act=True, res="sep"),
    bf(1, 1, 1, 1536, 768, 128, d=8, act=True),
    bf(1, 1, 3, 64, 32, 127, d=32, act=True),
    # conv_super_rows: C in {64, 512}, Cout = 2C; s 8 at C 512 is Cin 4096 (192 K steps)
    bf(1, 2, 3, 64, 128, 258, d=2, act=True),
    bf(1, 2, 1, 64, 128, 512, d=4, act=True),
    bf(1, 2, 1, 512, 1024, 2056, d=8, act=True),
    bf(1, 2, 3, 512, 1024, 254, d=2, raw=True, act=False),
]
GEN_GEOMS = [
    # (kind, B, Cin, Cout, T, taps, d, extra)
    (0, 3, 96, 48, 200, 7, 3, {}),
    (0, 2, 12, 6, 130, 7, 9, {"res": "sep"}),       # the tiny codec's widths, Cin < 16
    (0, 1, 6, 6, 20, 7, 9, {}),                     # dilation 9 at T < 27
    (0, 3, 24, 12, 70, 1, 1, {"res": "inplace"}),
    (0, 2, 6, 1, 100, 7, 1, {"tanh": True}),        # the final conv where final_conv_supported refuses (C % 8)
    (0, 1, 520, 1, 65, 7, 1, {"tanh": True}),       # ... and C > 512
    (0, 2, 1, 64, 300, 7, 1, {"samples": 250, "act": False}),   # the generic encode walk's input conv
    (1, 3, 96, 48, 65, 2, 8, {}),
    (1, 2, 24, 12, 33, 2, 4, {}),
    (1, 1, 12, 6, 40, 2, 2, {}),
    (1, 1, 64, 32, 9, 2, 32, {}),
    (2, 3, 16, 32, 256, 3, 4, {}),
    (2, 1, 64, 128, 258, 3, 2, {}),
    (2, 2, 8, 16, 64, 3, 8, {}),
]
GEN_CASES = [Case(0, dt, k, B, ci, co, T, taps, d, **{"act": True, **kw}) for dt in (BF, F32)
             for (k, B, ci, co, T, taps, d, kw) in GEN_GEOMS]
FINAL_CASES = [bf(2, 0, 3, 8, 1, 129, tanh=True), bf(2, 0, 1, 96, 1, 4097, tanh=True), bf(2, 0, 3, 160, 1, 127, tanh=True),
               bf(2, 0, 1, 512, 1, 128, tanh=True), bf(2, 0, 3, 96, 1, 1, tanh=True)]
INPUT_CASES = [bf(3, 0, 3, 1, 2, 128, samples=100, act=True), bf(3, 0, 1, 1, 64, 1024, samples=1000, act=True),
               bf(3, 0, 3, 1, 4096, 192, samples=130, act=True)]
RAGGED_CASES = [
    bf(1, 0, 4, 96, 96, 512, 7, 9, act=True, frames=8),
    bf(1, 0, 5, 64, 64, 1024, 7, 1, act=True, res="inplace", frames=4),
    bf(1, 1, 4, 128, 64, 32, d=4, act=True, frames=8),
    bf(2, 0, 4, 96, 1, 384, tanh=True, frames=6),
    Case(0, BF, 0, 4, 24, 12, 40, 7, 3, act=True, frames=5),
    Case(0, F32, 0, 4, 24, 12, 40, 7, 3, act=True, frames=5),
    Case(0, BF, 1, 4, 24, 12, 10, 2, 4, act=True, frames=5),
]
BENCH_CASE = bf(1, 0, 32, 96, 96, 248 * 512, 7, 9, raw=False, act=True, sample_rows=True)
SWEEP_CASES = [bf(1, 0, 2, 64, 64, 1024, 1, 1, act=True, sweep=True), bf(3, 0, 2, 1, 64, 2048, samples=2000, act=True, sweep=True),
               Case(0, BF, 0, 2, 64, 32, 1024, 1, 1, act=True, sweep=True)]


# ---- inputs ----------------------------------------------------------------------------------------------------------------
def make_inputs(c: Case, device="cpu") -> dict:
    """Model-dtype tensors of a case (float64 copies of what the kernel reads), PyTorch weight layouts."""
    g = torch.Generator().manual_seed(1000 + c.seed + 7 * c.Cin + 13 * c.Cout + c.T)
    k = 2 * c.d if c.kind else c.taps
    wshape = (c.Cin, c.Cout, k) if c.kind == 1 else (c.Cout, c.Cin, k)
    w = torch.randn(wshape, generator=g) / math.sqrt(c.cin_k * min(k, 7))
    w.view(-1)[torch.arange(3, w.numel(), 97)] *= 8.0                # outlier weights
    bias = torch.randn(c.Cout, generator=g) * 0.5
    if c.kernel == 3:
        x = torch.randn(c.B, c.tin, generator=g) * 0.5
    else:
        x = torch.randn(c.B, c.tin, c.Cin, generator=g)
        x[:, :, torch.arange(1, c.Cin, 11)] *= 6.0                   # outlier channels
        x *= torch.exp(torch.randn(c.B, c.tin, 1, generator=g) * 0.5)
    if c.sweep:   # rows of magnitude 2^-4 .. 2^6 and alpha over 2^-6 .. 2^6: |alpha x| covers 2^-10 .. 2^12
        if c.kernel == 3:
            x = x.sign() * torch.exp2(torch.empty(x.shape).uniform_(-4, 1, generator=g))
        else:
            x *= torch.exp2(torch.empty(c.B, c.tin, 1).uniform_(-4, 6, generator=g))
        bias *= torch.exp2(torch.empty(c.Cout).uniform_(-4, 9, generator=g)) if c.kernel == 3 else 8.0
        lo, hi = 2.0 ** -6, 2.0 ** 6
    else:
        lo, hi = c.alpha
    n_alpha = c.Cin if c.kernel == 0 else c.Cout

    def alpha():
        return torch.exp(torch.empty(n_alpha).uniform_(math.log(lo), math.log(hi), generator=g))
    d = dict(w=w, bias=bias, x=x, alpha=alpha() if c.act else None, alpha_own=alpha() if c.act else None)
    if c.res != "none":
        d["res"] = torch.randn(c.B, c.tout, c.Cout, generator=g) * 2.0
    if c.frames:
        d["lengths"] = torch.tensor(([0, 1, c.frames - 1, c.frames] + [c.frames // 2] * c.B)[:c.B], dtype=torch.int32)
        up_in, _ = c.up
        for b, n in enumerate(d["lengths"].tolist()):
            # the walks' invariant for the wgmma / final conv input: zeros over the band past the row's end (what the previous
            # conv wrote); finite garbage beyond it, which no kept output may read.  conv_kernel cuts the input at the end itself.
            e = n * up_in
            if c.kernel == 0:
                d["x"][b, e:] = 50.0
            else:
                d["x"][b, e:e + 129] = 0.0
                d["x"][b, e + 129:] = 50.0
    dt = c.dtype
    return {k2: (v.to(dt).double().to(device) if v.is_floating_point() else v.to(device)) if v is not None else None
            for k2, v in d.items()}


# ---- the reference ---------------------------------------------------------------------------------------------------------
def conv_f64(c: Case, x_cf: torch.Tensor, w: torch.Tensor, bug: str | None = None) -> torch.Tensor:
    """torch's conv of the case's kind over channels-first float64 input [B, Cin, Tin]."""
    k = w.shape[-1]
    if c.kind == 0:
        dil = 1 if bug == "dilation" else c.d
        pad = (k - 1) // 2 * dil
        if bug == "tap_offset":       # tap 0 reads one row further
            w0 = torch.zeros_like(w)
            w0[..., 0] = w[..., 0]
            xs = F.pad(x_cf[..., 1:], (0, 1))
            return F.conv1d(x_cf, w - w0, padding=pad, dilation=dil) + F.conv1d(xs, w0, padding=pad, dilation=dil)
        return F.conv1d(x_cf, w, padding=pad, dilation=dil)
    s = c.d
    if c.kind == 1:
        if bug == "phase_pad":        # o_add off by one: the transposed conv's padding one more
            y = F.conv_transpose1d(x_cf, w, stride=s, padding=math.ceil(s / 2) + 1)
            return F.pad(y, (0, x_cf.shape[-1] * s - y.shape[-1]))
        y = F.conv_transpose1d(x_cf, w, stride=s, padding=math.ceil(s / 2))
        if bug == "phase_mirror":     # output row q s - pad + p takes phase s - 1 - p
            pad = math.ceil(s / 2)
            yp = F.pad(y, (pad, s - pad))
            yp = yp.unflatten(-1, (-1, s)).flip(-1).flatten(-2)
            y = yp[..., pad:pad + y.shape[-1]]
        return y
    if bug == "super_row":            # tap r + j s - s/2 + 1: the window one input row earlier
        y = F.conv1d(F.pad(x_cf, (s // 2 + 1, s // 2 - 1)), w, stride=s)
        return y[..., :x_cf.shape[-1] // s]
    return F.conv1d(x_cf, w, stride=s, padding=s // 2)


@dataclasses.dataclass
class Ref:
    z: torch.Tensor              # conv + bias, fp64 [B, Tout, Cout]
    e: torch.Tensor              # E_acc
    res: torch.Tensor | None


def reference(c: Case, inp: dict, bug: str | None = None) -> dict:
    """Nearest values and candidate sets of the case's outputs ([B, Tout, Cout]; kernel 2: [B, T, 1])."""
    x, w, bias = inp["x"], inp["w"], inp["bias"]
    if c.kernel == 3:
        x = F.pad(x, (0, c.T - c.tin))[..., None]
    elif c.samples:
        x = F.pad(x, (0, 0, 0, c.T - c.tin))
    if c.frames:   # the reference of each row zero-padded past its end
        up_in, _ = c.up
        keep = torch.arange(x.shape[1], device=x.device)[None, :] < (inp["lengths"].to(x.device).long() * up_in)[:, None]
        x = x * keep[..., None]
    if bug == "batch":
        x = torch.cat([x[:1], x[:-1]])
    if bug == "cin_chunk":           # the last K chunk (64 channels wgmma, 16 generic) dropped
        ck = 64 if c.kernel == 1 else 16
        if c.kind == 2:
            xs = x.reshape(c.B, x.shape[1] // c.d, c.d * c.Cin).clone()
            xs[..., (c.cin_k - 1) // ck * ck:] = 0
            x = xs.reshape(x.shape)
        else:
            x = x.clone()
            x[..., (c.Cin - 1) // ck * ck:] = 0
    spread = None
    out = {}
    if c.kernel == 0 and c.act:      # snake on the input, per channel
        a = inp["alpha"]
        if c.dtype == BF:
            near, lo, hi, amb, axa = snake_set(x, a, inv_of(a))
            spread = hi - lo
            out["sin_amb_in"] = int(amb.sum())
            out["ax_max"] = float(axa.max())
            x_act, delta = near, None
        else:
            inv = 1.0 / (a + 1e-9)
            ax = a * x
            t = inv * torch.sin(ax) ** 2
            x_act = x + t
            delta = 12 * U * t + (torch.sin(2 * ax).abs() * ax.abs() * U) * inv + U * x_act.abs()
            spread = delta
            out["ax_max"] = float(ax.abs().max())
    else:
        x_act = x
    x_cf = x_act.permute(0, 2, 1)
    z = conv_f64(c, x_cf, w, bug).permute(0, 2, 1) + bias
    mass = conv_f64(c, x_cf.abs(), w.abs()).permute(0, 2, 1)
    e = U * (c.n_chain + 32) * mass + U * z.abs()
    if spread is not None:
        e = e + conv_f64(c, spread.permute(0, 2, 1), w.abs()).permute(0, 2, 1)
    res = inp.get("res")
    if bug == "residual":
        res = None
    out.update(z=z, e=e, mass=mass)
    if c.dtype == F32:
        ref = z if res is None else z + res
        bar = e + 4 * U * (ref.abs() + (res.abs() if res is not None else 0))
        if c.tanh and bug != "tanh":
            ref = torch.tanh(ref)
            bar = bar + 2 * ulp_f32(ref)
        out.update(ref=ref, bar=bar)
        return _ragged_ref(c, inp, out, bug)
    r_near, r_lo, r_hi = rn(z), rn(z - e), rn(z + e)
    out["raw_amb"] = bf_ord(r_hi) > bf_ord(r_lo)
    if res is not None:
        r_near, r_lo, r_hi = rn(res + r_near), rn(res + r_lo), rn(res + r_hi)
    out.update(raw=r_near, raw_lo=r_lo, raw_hi=r_hi)
    if c.tanh:
        if bug == "tanh":
            out.update(ref=r_near, lo=r_lo, hi=r_hi)
        else:
            t_lo, t_hi = tanh_set(r_lo, r_hi)
            out.update(ref=rn(torch.tanh(r_near)), lo=t_lo, hi=t_hi)
    if c.kernel in (1, 3) and c.act:
        a = inp["alpha_own"] if bug == "alpha_own" else inp["alpha"]
        inv = inv_of(a)
        if bug == "inv_unrounded":
            inv = 1.0 / (a.float() + 1e-9).bfloat16().double()
        near, _, _, amb, axa = snake_set(r_near, a, inv)
        if bug == "sin_not_squared":
            near = rn(r_near + rn(inv * rn(torch.sin(rn(a * r_near)))))
        out.update(act=near, sin_amb=amb, ax_max=float(axa.max()), act_inv=inv, act_alpha=a)
    return _ragged_ref(c, inp, out, bug)


def _ragged_ref(c, inp, out, bug):
    if bug == "tile_row" or bug == "final_shift":
        for k in ("ref", "raw", "act", "z"):
            if k in out and out[k] is not None:
                v = out[k].clone()
                if bug == "tile_row":
                    v[:, 127::128] = 0.0
                else:
                    v[:, :-1] = out[k][:, 1:]
                out[k] = v
    if bug == "n_tile":
        for k in ("ref", "raw", "act", "z"):
            if k in out:
                v = out[k].clone()
                v[..., (c.Cout - 1) // 32 * 32:] = 0.0
                out[k] = v
    return out


def act_member(got: torch.Tensor, out: dict, e_k: int = 8):
    """Is each act value a member of the candidate set (any raw candidate, either sin neighbour where ambiguous)?"""
    lo_o, hi_o = bf_ord(out["raw_lo"]), bf_ord(out["raw_hi"])
    n = int((hi_o - lo_o).max()) + 1
    ok = torch.zeros_like(got, dtype=torch.bool)
    g = bf_ord(got)
    for k in range(min(n, e_k)):
        r = bf_from_ord(torch.minimum(lo_o + k, hi_o))
        _, lo, hi, _, _ = snake_set(r, out["act_alpha"], out["act_inv"])
        ok |= (g >= bf_ord(lo)) & (g <= bf_ord(hi))
    if n > e_k:   # a raw interval of more than e_k values (a sum that cancels to near 0): snake(r) lies in [r, r + inv]
        lo, hi = out["raw_lo"], out["raw_hi"] + out["act_inv"]
        ok |= (hi_o - lo_o >= e_k) & (got >= lo - 2.0 ** -7 * lo.abs()) & (got <= hi + 2.0 ** -7 * hi.abs())
    return ok


# ---- running a case ----------------------------------------------------------------------------------------------------------
def scratch_bytes(c: Case) -> int:
    k = 2 * c.d if c.kind else c.taps
    return (2 * c.Cin * c.Cout * k + k * c.Cin) * 4 + 256


def run_case(c: Case, inp: dict, pad: int = 3):
    """The hook on device copies of the case's inputs; outputs [B * Tout + pad, Cout] start as NaN."""
    from parler_tts_b200 import _lib
    dt = c.dtype
    dev = {k: (v.to(dt).to(DEV).contiguous() if v.is_floating_point() else v.to(DEV).contiguous()) if v is not None else None
           for k, v in inp.items()}
    rows = c.B * c.tout
    nan = float("nan")
    out_raw = torch.full((rows + pad, c.Cout), nan, dtype=dt, device=DEV) if c.raw or c.kernel != 1 else None
    out_act = torch.full((rows + pad, c.Cout), nan, dtype=dt, device=DEV) if c.act and c.kernel in (1, 3) else None
    res = None
    if c.res == "sep":
        res = dev["res"]
    elif c.res == "inplace":
        out_raw[:rows] = dev["res"].reshape(rows, c.Cout)
        res = out_raw
    scratch = torch.empty(scratch_bytes(c), dtype=torch.uint8, device=DEV)
    a_in = dev["alpha"] if c.kernel == 0 and c.act else None
    a_next = dev["alpha"] if c.kernel in (1, 3) and c.act else None
    fl = dev.get("lengths")
    _lib.check(_lib.lib().ptts_op_dac_conv(
        _lib.dtype_code(dt), c.kernel, c.kind, c.B, c.Cin, c.Cout, c.T, c.taps, c.d, c.samples, _lib.ptr(dev["w"]),
        _lib.ptr(dev["bias"]), _lib.ptr(a_in), _lib.ptr(a_next), _lib.ptr(dev["x"]), _lib.ptr(res), _lib.ptr(out_raw),
        _lib.ptr(out_act), int(c.tanh), _lib.ptr(fl), c.frames, _lib.ptr(scratch), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return out_raw, out_act


def select_rows(c: Case) -> torch.Tensor:
    """Output rows compared on a large shape: the first and last 128-row tiles, both sides of every tile edge, 256 random."""
    T = c.tout
    edges = torch.arange(128, T, 128)
    rows = torch.cat([torch.arange(0, 128), torch.arange(max(0, (T - 1) // 128 * 128), T), edges - 1, edges,
                      torch.randint(0, T, (256,), generator=torch.Generator().manual_seed(5))])
    return torch.unique(rows.clamp(0, T - 1))


def reference_rows(c: Case, inp: dict, rows: torch.Tensor) -> dict:
    """The reference at selected output rows of a conv_same case: F.conv1d over each row's zero-padded input window."""
    x = inp["x"]
    k, dil = c.taps, c.d
    pad = (k - 1) // 2 * dil
    out = {}
    bsel = [0, c.B // 2, c.B - 1]
    xs = []
    for b in bsel:
        xp = F.pad(x[b].T[None], (pad, pad))[0]                      # [Cin, T + 2 pad]
        idx = rows.to(x.device)[:, None] + torch.arange(0, (k - 1) * dil + 1, device=x.device)[None, :]
        xs.append(xp[:, idx].permute(1, 0, 2))                        # [R, Cin, window]
    win = torch.cat(xs).double()
    sub = dataclasses.replace(c, B=len(bsel) * len(rows), T=(k - 1) * dil + 1, sample_rows=False)
    ref = reference(sub, dict(inp, x=win.permute(0, 2, 1).contiguous()))
    mid = (k - 1) // 2 * dil                                          # the window's centre row is the output row
    for key in ("raw", "raw_lo", "raw_hi", "act", "sin_amb", "raw_amb", "z", "e"):
        if key in ref:
            ref[key] = ref[key][:, mid:mid + 1].reshape(len(bsel), len(rows), -1)
    ref["bsel"] = bsel
    return ref


def check_case(c: Case):
    inp = make_inputs(c, DEV)
    out_raw, out_act = run_case(c, inp)
    rows = c.B * c.tout
    tag = (c.kernel, "bf16" if c.dtype == BF else "f32")
    st = STATS.setdefault(tag, [0, 0, 0, 0, 0.0])
    st[0] += 1
    for o, name in ((out_raw, "out_raw"), (out_act, "out_act")):
        if o is not None:
            assert torch.isnan(o[rows:].float()).all(), f"{c.id}: {name} rows past B * Tout were written"
    if c.sample_rows:
        sel = select_rows(c)
        ref = reference_rows(c, inp, sel.to(DEV))
        got_act = out_act[:rows].view(c.B, c.tout, c.Cout)[ref["bsel"]][:, sel.to(DEV)].double()
        assert not torch.isnan(got_act).any(), f"{c.id}: out_act not written"
        _check_act(c, got_act, ref, st)
        st[1] += got_act.numel()
        return
    ref = reference(c, inp)
    shape = (c.B, c.tout, c.Cout)
    got_raw = out_raw[:rows].view(shape).double() if out_raw is not None else None
    got_act = out_act[:rows].view(shape).double() if out_act is not None else None
    keep = torch.ones(shape[:2], dtype=torch.bool, device=DEV)
    if c.frames:
        _, up_out = c.up
        end = inp["lengths"].long()[:, None] * up_out
        t = torch.arange(c.tout, device=DEV)[None, :]
        keep = t < end
        band = (t >= end) & (t < end + 129)
        for g, name in ((got_raw, "out_raw"), (got_act, "out_act")):
            if g is None:
                continue
            past = g[~keep]
            if c.kernel == 1:   # the zero band exactly 0; later tiles may be left unwritten, never given anything else
                assert (g[band] == 0).all(), f"{c.id}: {name} not 0 over the zero band past a row's end"
                before = inp["res"][~keep] if (name == "out_raw" and c.res == "inplace") else torch.full_like(past, float("nan"))
                unwritten = torch.isnan(past) if name == "out_act" or c.res != "inplace" else past == before
                assert ((past == 0) | unwritten).all(), f"{c.id}: {name} past a row's end is neither 0 nor unwritten"
            else:
                assert (past == 0).all(), f"{c.id}: {name} not exactly 0 past a row's end"
    for g, name in ((got_raw, "out_raw"), (got_act, "out_act")):
        if g is not None:
            assert not torch.isnan(g[keep]).any(), f"{c.id}: {name} has unwritten elements inside the shape"
    m = keep[..., None].expand(shape)
    st[1] += int(m.sum()) * (int(got_raw is not None) + int(got_act is not None))
    if c.dtype == F32:
        ratio = ((got_raw - ref["ref"]).abs() / ref["bar"])[m]
        worst = float(ratio.max())
        st[4] = max(st[4], worst)
        if worst > 1.0:
            i = int(ratio.argmax())
            raise AssertionError(f"{c.id}: |got - ref| = {worst:.2f} x bar at element {i}: got {float(got_raw[m][i])!r} "
                                 f"ref {float(ref['ref'][m][i])!r} ({int((ratio > 1).sum())} over)")
        return
    st[2] += int(ref["raw_amb"][m].sum())
    if c.tanh:
        _member(c, "out_raw (tanh)", got_raw, ref["lo"], ref["hi"], ref["ref"], m)
    elif got_raw is not None:
        _member(c, "out_raw", got_raw, ref["raw_lo"], ref["raw_hi"], ref["raw"], m)
    if c.kernel == 0 and c.act:
        st[3] += ref["sin_amb_in"]
        _sweep(c, ref["ax_max"], ref["sin_amb_in"])
    if got_act is not None:
        _check_act(c, got_act, ref, st, m)


def _member(c, what, got, lo, hi, near, m):
    ok = (bf_ord(got) >= bf_ord(lo)) & (bf_ord(got) <= bf_ord(hi))
    bad = ~ok & m
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{c.id}: {what} outside its candidate set at {i}: got {float(got[tuple(i)])!r}, "
                             f"set [{float(lo[tuple(i)])!r}, {float(hi[tuple(i)])!r}], nearest {float(near[tuple(i)])!r} "
                             f"({int(bad.sum())} elements)")


def _check_act(c, got_act, ref, st, m=None):
    st[3] += int(ref["sin_amb"].sum() if m is None else ref["sin_amb"][m].sum())
    _sweep(c, ref["ax_max"], int(ref["sin_amb"].sum()))
    ok = act_member(got_act, ref)
    bad = ~ok if m is None else (~ok & m)
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{c.id}: out_act outside its candidate set at {list(i)}: got {float(got_act[i])!r}, nearest "
                             f"{float(ref['act'][i])!r} from raw {float(ref['raw'][i])!r}, alpha "
                             f"{float(ref['act_alpha'][i[-1]])!r} ({int(bad.sum())} elements)")


def _sweep(c, ax_max, amb):
    if c.sweep:
        s = SWEEP.setdefault(c.kernel, [0.0, 0])
        s[0] = max(s[0], ax_max)
        s[1] += amb


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    for (k, dt), (n, el, raw2, sin2, worst) in sorted(STATS.items()):
        print(f"\n[dac conv reference] kernel {k} {dt}: {n} cases, {el} elements, {raw2} with two raw candidates, "
              f"{sin2} with two sin candidates" + (f", worst f32 error / bar {worst:.3f}" if dt == "f32" else ""))
    for k, (ax, amb) in sorted(SWEEP.items()):
        print(f"\n[dac conv reference] snake sweep, kernel {k}: |alpha x| up to {ax:.4g}, {amb} elements with two sin candidates")


# ---- GPU tests -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("c", TC_CASES, ids=lambda c: c.id)
def test_conv_tc_kernel(c):
    check_case(c)


@pytest.mark.gpu
@pytest.mark.parametrize("c", GEN_CASES, ids=lambda c: c.id)
def test_conv_kernel(c):
    check_case(c)


@pytest.mark.gpu
@pytest.mark.parametrize("c", FINAL_CASES + INPUT_CASES, ids=lambda c: c.id)
def test_final_and_input_conv(c):
    check_case(c)


@pytest.mark.gpu
@pytest.mark.parametrize("c", RAGGED_CASES, ids=lambda c: c.id)
def test_ragged(c):
    check_case(c)


@pytest.mark.gpu
def test_bench_sized_launch():
    """The last decoder block's k7 dil-9 conv of the 44.1 kHz codec at the bench's batch: B = 32 x 248 frames, 96 channels."""
    check_case(BENCH_CASE)


@pytest.mark.gpu
@pytest.mark.parametrize("c", SWEEP_CASES, ids=lambda c: c.id)
def test_snake_large_arguments(c):
    """snake where |alpha x| spans 2^-10 .. 2^12: sin must round like the correctly rounded value, not like an approximation
    whose error grows with the argument."""
    check_case(c)


@pytest.mark.gpu
def test_refusals():
    from parler_tts_b200 import _lib
    x, o, scr = (torch.zeros(1 << 16, dtype=torch.bfloat16, device=DEV) for _ in range(3))
    fl = torch.tensor([1, 2], dtype=torch.int32, device=DEV)
    p = _lib.ptr(x)

    def call(dtype=_lib.BF16, kernel=0, kind=0, B=1, Cin=64, Cout=64, T=64, taps=7, d=1, samples=0, alpha=None,
             alpha_next=None, out_act=None, tanh=0, lengths=None, frames=0):
        return _lib.check(_lib.lib().ptts_op_dac_conv(dtype, kernel, kind, B, Cin, Cout, T, taps, d, samples, p, p, alpha,
                                                      alpha_next, p, None, _lib.ptr(o), out_act, tanh, lengths, frames,
                                                      _lib.ptr(scr), _lib.stream_ptr()))
    call()                                                       # a valid launch
    cases = [dict(taps=9), dict(d=11),                           # launch_conv: taps > 7, receptive field past its tile
             dict(kernel=1, d=43, B=2, T=128, lengths=_lib.ptr(fl), frames=2),   # a ragged reach past the 128-row zero band
             dict(kernel=1, dtype=_lib.F32), dict(kernel=1, Cout=48), dict(kernel=1, Cin=32), dict(kernel=1, Cin=100),
             dict(kernel=1, alpha=p), dict(kernel=1, out_act=p),
             dict(kernel=2, Cout=1, Cin=12, tanh=1), dict(kernel=2, Cout=1, Cin=520, tanh=1), dict(kernel=2, Cout=2, tanh=1),
             dict(kernel=3, Cin=2, samples=10, alpha_next=p, out_act=p), dict(kernel=3, Cin=1, samples=0, alpha_next=p, out_act=p),
             dict(kernel=0, alpha_next=p), dict(kind=1, d=3), dict(kind=2, d=4, T=66), dict(kernel=4), dict(dtype=2)]
    for kw in cases:
        with pytest.raises(ValueError):
            call(**kw)
    torch.cuda.synchronize()


# ---- host tests --------------------------------------------------------------------------------------------------------------
def test_hook_is_bound():
    from parler_tts_b200 import _lib
    assert "ptts_op_dac_conv" in _lib._SIGS and len(_lib._SIGS["ptts_op_dac_conv"][1]) == 23


def _seen(c: Case, ref: dict, bad: dict) -> float:
    """How far the bug's reference lies outside the case's bar, at its worst element: f32, |bad - ref| / bar; bf16, the distance
    in bf16 values from the candidate set (the bug is seen at 2, where even a member check with one extra neighbour fails)."""
    if c.dtype == F32:
        d = (bad["ref"] - ref["ref"]).abs() / ref["bar"]
        return float(torch.where(torch.isnan(d), torch.zeros_like(d), d).max())
    if "act" in ref:
        v = bad["act"]
        o = bf_ord(v)
        inside = act_member(v, ref)
        near = inside | act_member(bf_from_ord(o + 1), ref) | act_member(bf_from_ord(o - 1), ref)
        return 0.0 if inside.all() else 1.0 if near.all() else 2.0
    v, lo, hi = (bad["ref"], ref["lo"], ref["hi"]) if "lo" in ref else (bad["raw"], ref["raw_lo"], ref["raw_hi"])
    o = bf_ord(v)
    return float(torch.maximum(bf_ord(lo) - o, o - bf_ord(hi)).clamp(min=0).max())


SENSITIVITY = [
    ("tap_offset", bf(1, 0, 2, 64, 32, 40, 7, 3, act=True)),
    ("tap_offset", Case(0, F32, 0, 2, 12, 6, 40, 7, 9, act=True)),
    ("dilation", bf(1, 0, 2, 64, 32, 40, 7, 9, act=True)),
    ("phase_mirror", bf(1, 1, 2, 64, 32, 12, d=4, act=True)),
    ("phase_pad", bf(1, 1, 2, 64, 32, 12, d=8, act=True)),
    ("phase_mirror", Case(0, F32, 1, 2, 12, 6, 10, 2, 2, act=True)),
    ("super_row", bf(1, 2, 2, 64, 128, 32, d=4, act=True)),
    ("super_row", Case(0, BF, 2, 2, 8, 16, 32, 3, 2, act=True)),
    ("cin_chunk", bf(1, 0, 2, 96, 32, 40, 7, 1, act=True)),
    ("cin_chunk", bf(1, 2, 1, 64, 128, 32, d=2, raw=True, act=False)),
    ("cin_chunk", Case(0, BF, 0, 2, 24, 12, 40, 7, 1, act=True)),
    ("tile_row", bf(1, 0, 1, 64, 32, 200, 7, 1, act=True)),
    ("n_tile", bf(1, 0, 1, 64, 160, 40, 7, 1, act=True)),
    ("batch", bf(1, 0, 3, 64, 32, 40, 7, 1, act=True)),
    ("residual", bf(1, 0, 2, 64, 32, 40, 7, 1, act=True, res="sep")),
    ("residual", Case(0, F32, 0, 2, 12, 6, 40, 7, 1, act=True, res="inplace")),
    ("alpha_own", bf(1, 0, 2, 64, 32, 40, 7, 1, act=True)),
    ("alpha_own", bf(3, 0, 2, 1, 64, 64, samples=60, act=True)),
    ("sin_not_squared", bf(1, 0, 2, 64, 32, 40, 7, 1, act=True)),
    ("inv_unrounded", bf(1, 0, 2, 64, 32, 40, 7, 1, act=True)),
    ("tanh", bf(2, 0, 2, 96, 1, 40, tanh=True)),
    ("tanh", Case(0, F32, 0, 2, 6, 1, 40, 7, 1, act=True, tanh=True)),
    ("final_shift", bf(2, 0, 2, 96, 1, 40, tanh=True)),
]


@pytest.mark.parametrize("bug,c", SENSITIVITY, ids=[f"{b}-{c.id}" for b, c in SENSITIVITY])
def test_sensitivity(bug, c):
    """Each modelled kernel bug moves its case's reference past the bar on some element: by more than 4x the f32 bar, or to at
    least two bf16 values outside the candidate set."""
    inp = make_inputs(c)
    seen = _seen(c, reference(c, inp), reference(c, inp, bug))
    ok = seen > 4.0 if c.dtype == F32 else seen >= 2.0
    assert ok, f"{bug} moves {c.id} by only {seen:.2f}"


@pytest.mark.parametrize("c", [Case(0, F32, 0, 2, 24, 12, 50, 7, 3, act=True, res="sep"), Case(0, F32, 1, 2, 24, 12, 20, 2, 4, act=True),
                               Case(0, F32, 2, 2, 16, 32, 64, 3, 4, act=True), Case(0, F32, 0, 2, 8, 1, 50, 7, 1, act=True, tanh=True)],
                         ids=lambda c: c.id)
def test_reference_matches_torch_f32(c):
    """With f32 inputs the reference is torch's fp32 layer (snake, conv, bias, residual, tanh) within the f32 bar."""
    from oracle.dac import snake
    inp = make_inputs(c)
    ref = reference(c, inp)
    x = snake(inp["x"].float(), inp["alpha"].float()).permute(0, 2, 1)
    w, b = inp["w"].float(), inp["bias"].float()
    if c.kind == 0:
        y = F.conv1d(x, w, b, padding=(c.taps - 1) // 2 * c.d, dilation=c.d)
    elif c.kind == 1:
        y = F.conv_transpose1d(x, w, b, stride=c.d, padding=math.ceil(c.d / 2))
    else:
        y = F.conv1d(x, w, b, stride=c.d, padding=c.d // 2)
    y = y.permute(0, 2, 1).double()
    if c.res != "none":
        y = (y.float() + inp["res"].float()).double()
    if c.tanh:
        y = torch.tanh(y.float()).double()
    err = ((y - ref["ref"]).abs() / ref["bar"]).max()
    assert float(err) <= 1.0, f"torch fp32 differs from the reference by {float(err):.2f}x the bar"


def test_reference_contains_bf16_oracle():
    """With bf16 inputs, OracleDAC(..., torch.bfloat16)'s layers on the CPU are members of the reference's candidate sets: the
    transposed conv of a decoder block (snake on its input), a residual unit's k7 dil-3 conv, and the final conv + tanh."""
    from oracle.config import tiny_dac_cfg
    from oracle.dac import OracleDAC, snake
    from oracle.weights import make_dac_weights
    cfg = tiny_dac_cfg()
    o = OracleDAC(cfg, make_dac_weights(cfg, seed=3), torch.bfloat16)
    g = torch.Generator().manual_seed(11)
    p = "decoder.block.0."
    layers = [  # (case, weight key, bias key, alpha key, oracle fn)
        (Case(0, BF, 1, 2, 96, 48, 24, 2, 8, act=True), p + "conv_t1.weight", p + "conv_t1.bias", p + "snake1.alpha",
         lambda x, w, b: F.conv_transpose1d(x, w, b, stride=8, padding=4)),
        (Case(0, BF, 0, 2, 48, 48, 60, 7, 3, act=True), p + "res_unit2.conv1.weight", p + "res_unit2.conv1.bias",
         p + "res_unit2.snake1.alpha", lambda x, w, b: F.conv1d(x, w, b, dilation=3, padding=9)),
        (Case(0, BF, 0, 2, 6, 1, 60, 7, 1, act=True, tanh=True), "decoder.conv2.weight", "decoder.conv2.bias", "decoder.snake1.alpha",
         lambda x, w, b: torch.tanh(F.conv1d(x, w, b, padding=3))),
    ]
    for c, wk, bk, ak, fn in layers:
        x = torch.randn(c.B, c.Cin, c.T, generator=g).bfloat16()
        got = fn(snake(x, o.w[ak]), o.w[wk], o.w[bk]).permute(0, 2, 1).double()
        inp = dict(x=x.permute(0, 2, 1).double(), w=o.w[wk].double(), bias=o.w[bk].double(), alpha=o.w[ak].reshape(-1).double())
        ref = reference(c, inp)
        lo, hi = (ref["lo"], ref["hi"]) if c.tanh else (ref["raw_lo"], ref["raw_hi"])
        ok = (bf_ord(got) >= bf_ord(lo)) & (bf_ord(got) <= bf_ord(hi))
        assert ok.all(), f"{c.id}: {int((~ok).sum())} oracle values outside the candidate sets"


def test_candidate_helpers():
    """bf_ord / bf_from_ord walk adjacent bf16 values; snake_set's set holds the nearest value."""
    v = torch.tensor([-3.0, -1e-3, 0.0, 1e-30, 1.0, 2.5e4]).double()
    v = rn(v)
    o = bf_ord(v)
    assert torch.equal(bf_from_ord(o), v)
    nxt = bf_from_ord(o + 1)
    mid = rn((v + nxt) / 2)
    assert (nxt > v).all() and ((mid == v) | (mid == nxt)).all()
    r = rn(torch.linspace(-40, 40, 4001).double())[:, None]
    a = rn(torch.tensor([0.013, 0.7, 3.1, 95.0]).double())
    near, lo, hi, _, _ = snake_set(r, a, inv_of(a))
    assert ((near >= lo) & (near <= hi)).all()
