"""The codec's quantizer kernels one launch at a time, against a float64 reference, through the ptts_op_dac_quantize and
ptts_op_dac_from_codes hooks.

quantize_kernel (dac_enc.cu) is the residual vector quantizer of DACModel.encode: one warp per code frame, lane l owning latent
channels l, l + 32, ...; per codebook e = rn(in_proj(r) + b) (lane-strided fmaf chains, a 5-level butterfly, the bias add), the
cosine of e / |e| against fp32 unit rows (packed by pack_normalized_codebook, the rows rounded to bf16 first in a bf16 model),
a lane-strided argmax with ties to the lowest index, st = rn(e + rn(zq - e)), q = rn(out_proj(st) + b_out) and r = rn(r - q).
from_codes_kernel (dac.cu) turns codes into latents: rn(sum_d w c + b) per codebook, accumulated as acc = rn(acc + s) from
k = 0, as quantized_representation += ... does in the model dtype.  rn is one rounding to bf16 (the identity in an f32 model);
u = 2^-24.  Every bar below comes from the arithmetic, none from a run.

Quantizer reference: float64 along the kernel's own codes, one codebook at a time, over a set of states per frame.  A state is
one st history: a residual box [lo, hi] of bf16 values per element, holding every residual the kernel can reach on it (the q
roundings are independent per element, so the box is exact for them), and its nearest path inside it.
  e:     the bf16 vectors in [rn(e_lo - E_e), rn(e_hi + E_e)], e_lo / e_hi = in_proj over the residual box + b in float64 and
         E_e = (ceil(Z/32) + 6) u M + u (M + |b|), M = sum |w| max|r|: ceil(Z/32) chained fmaf per lane, 5 butterfly levels and
         one spare order each err by at most u M; the bias add by u |sum + b|.  Every point of that box is enumerated, except
         in an element whose range holds more than FINE values (it lies near 0, where bf16 values are dense), and in the
         widest elements of a box that would still hold more than CAP points: such an element is held at its nearest value and the pick gets 4 |width| / |e| of slack, width the norm of those elements' ranges (a
         cosine moves by at most 2 |delta| / |e|); st is still taken over the element's whole range.  Where that range gives
         more than FINE distinct st values the frame is no longer followed, and its later picks are counted as unfollowed.
  pick:  passes when, for some point e of the box, cos(e, c_pick) >= max_j cos(e, c_j) - 2 E_sim, with no lower index whose
         unit row is bit-identical to the pick's (exact ties go to the lowest index) and code 0 when e is exactly 0.  E_sim =
         (2 D + 8) u bounds the kernel's fp32 similarity: |e| and the row norms are D-term fmaf sums (D u relative), then sqrt,
         1/x and the scaling add 3 u: each unit vector is off by (D/2 + 3) u per element relative, and the D-term dot product of
         two of them by D u more.  1.4e-6 at D = 8.
  st:    rn(e + rn(zq - e)) of every accepted point, exactly as fp32 then bf16 computes it (elementwise in e); each distinct st
         vector starts a state of its own.
  q:     rn(q64 +- E_q), q64 = out_proj(st) + b in float64 and E_q = (D + 1) u M_q + u (M_q + |b|), M_q = sum |w| |st|.
  r:     [rn(r_lo - q_hi), rn(r_hi - q_lo)] (fp32 subtraction then bf16, monotone), with the nearest path inside it.
         More than SCAP states in a frame are merged into one holding their union (sound, looser), and counted.
  f32 model: the same chain with no roundings; r carries an absolute bound, e's error E_e moves each cosine by at most
  2 |E_e| / |e|, so a pick passes within 2 E_sim + 4 |E_e| / |e| of the best; st = zq within 3 u (|zq| + |e| + |E_e|), q within
  (D + 1) u M_q + sum |w| d_st + u |q|, r within d_r + d_q + u |r|.
  Reported per (dtype): picks; picks that needed any slack, and those that needed more than 2 E_sim (a near-0 element's);
  picks that needed an ambiguous-rounding branch (the nearest path refused them); undecided picks, whose slack reaches the gap
  between the two best similarities, so that the check could not tell the runner-up from the best; merged frames; the most
  box points and states in a frame; the worst gap / (2 E_sim), or gap / slack in f32.  A real-shape host test holds the check
  to catching the runner-up at the last codebook in nearly every frame.

from_codes reference: s64 = sum_d w c + b per codebook in float64 with E_s = (D + 1) u sum |w c| + u |s64|.  bf16: each s is a
value of [rn(s64 - E_s), rn(s64 + E_s)] and the sum's interval is [rn(acc_lo + s_lo), rn(acc_hi + s_hi)] per step (the conv
test's member check); the output must lie in it.  f32: |got - ref| <= sum_k (E_s,k + u |acc_k|).

Invariants on every launch: buffers start as NaN (codes as -7) with a tail past B * T that must stay so; every frame inside the
shape is written except the frames a window leaves alone on purpose; two launches give the same bits.  Ragged quantize: frames at
or past F_b = ceil(clamp(n_b, 1, T hop) / hop) hold code codebook_size and a zero latent, earlier frames the codes of the
non-ragged launch.  A NaN latent frame codes 0 in every codebook and leaves its neighbours as they are.  The packed unit rows
lie within (D/2 + 3) u |ref| of the float64 normalisation.

Host tests: the reference with every rounding off reproduces OracleDACEncoder.quantize in float64 and the fixture's codes where
its margin is clear; from_codes' reference matches OracleDAC.from_codes; a simulated kernel (nearest roundings) passes; and each
modelled kernel bug fails two or more picks or values, or moves an f32 value past 4x its bar.  One bug is not modelled: e
without the normalisation scales every similarity of a frame by |e|, which leaves the argmax where it was.
"""
from __future__ import annotations

import dataclasses
import math
import os

import numpy as np
import pytest
import torch

from tests.test_dac_conv_reference import bf_from_ord, bf_ord, rn

U = 2.0 ** -24
DEV = "cuda"
BF, F32 = torch.bfloat16, torch.float32
CAP = 1024
QSTATS: dict = {}    # dtype -> dict of summed counts and maxima (check_codes' keys)
FSTATS: dict = {}    # dtype -> [cases, values, values with two candidates, worst error / bar]


def dtn(dt):
    return "bf16" if dt == BF else "f32"


def model(t: torch.Tensor, dt) -> torch.Tensor:
    """A float64 tensor as the model dtype holds it (torch.float64: as it is, every rounding off)."""
    return rn(t) if dt == BF else t.float().double() if dt == F32 else t


# ---- quantizer cases -------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class QCase:
    dtype: torch.dtype
    D: int
    Z: int
    cs: int
    n_q: int
    B: int
    T: int
    kind: str = "random"        # random, dup, zero_rows, zero_e
    nan_frame: int = -1
    ragged: int = 0             # > 0: the hop of a ragged launch
    seed: int = 0

    @property
    def id(self):
        s = f"{dtn(self.dtype)}-D{self.D}-Z{self.Z}-cs{self.cs}-nq{self.n_q}-B{self.B}T{self.T}"
        if self.kind != "random":
            s += "-" + self.kind
        if self.nan_frame >= 0:
            s += "-nan"
        if self.ragged:
            s += f"-ragged{self.ragged}"
        return s


def _qcases(dt):
    Q = lambda *a, **k: QCase(dt, *a, **k)   # noqa: E731
    return [
        Q(4, 1, 33, 32, 1, 7),                   # Z = 1; the largest n_q for D = 4
        Q(8, 31, 1, 9, 1, 8),                    # cs = 1: every lane but 0 without a row
        Q(8, 32, 2, 1, 1, 1),
        Q(16, 33, 31, 16, 3, 3),                 # the largest n_q for D = 16
        Q(8, 1000, 32, 9, 1, 9),
        Q(16, 1024, 1024, 9, 2, 4),
        Q(4, 1536, 4096, 9, 3, 3),               # 8 warps x 1536 x 4 B = 48 KB of dynamic shared memory
        Q(8, 1536, 33, 32, 1, 9),                # the largest n_q for D = 8
        Q(4, 1024, 32, 1, 1, 8),
        Q(8, 64, 1024, 4, 2, 16, kind="dup"),
        Q(4, 64, 40, 3, 1, 20, kind="dup", seed=1),
        Q(16, 32, 2, 3, 1, 16, kind="zero_rows"),
        Q(8, 40, 33, 3, 1, 9, kind="zero_rows", seed=1),
        Q(8, 33, 31, 3, 1, 9, kind="zero_e"),
        Q(8, 100, 64, 9, 2, 5, nan_frame=6),
    ]


Q_CASES = _qcases(BF) + _qcases(F32)
Q_RAGGED = [QCase(BF, 8, 64, 64, 9, 8, 5, ragged=4), QCase(F32, 4, 33, 33, 3, 8, 3, ragged=7)]
Q_REAL = QCase(BF, 8, 1024, 1024, 9, 32, 173)


def make_q(c: QCase) -> dict:
    """Source weights (fp32, PyTorch layouts stacked over codebooks) and latents [B*T, Z] in the model dtype, float64."""
    g = torch.Generator().manual_seed(100 + c.seed + c.D * 7 + c.Z + c.cs * 3 + c.n_q)
    D, Z, cs, n_q = c.D, c.Z, c.cs, c.n_q
    w = dict(in_w=torch.randn(n_q, D, Z, generator=g) / math.sqrt(Z), in_b=torch.randn(n_q, D, generator=g) * 0.1,
             cb=torch.randn(n_q, cs, D, generator=g), out_w=torch.randn(n_q, Z, D, generator=g) / math.sqrt(D),
             out_b=torch.randn(n_q, Z, generator=g) * 0.05)
    w = {k: v.double() for k, v in w.items()}
    z = torch.randn(c.B * c.T, Z, generator=g, dtype=torch.float64) * 0.5
    if c.kind == "dup":      # row j's duplicates (exact, or scaled by a power of two) at j + 1, j + 31 .. j + 33 and cs - 1
        j = 3
        for i, s in ((j + 1, 1.0), (j + 31, 2.0), (j + 32, 0.5), (j + 33, 1.0), (cs - 1, 4.0)):
            w["cb"][:, i] = w["cb"][:, j] * s
        # latents whose first e points at row j: its whole group ties at the top
        W0, b0 = model(w["in_w"][0], c.dtype), model(w["in_b"][0], c.dtype)
        tgt = model(w["cb"][0, j], c.dtype) * 1.5 - b0
        z[::2] = (torch.linalg.pinv(W0) @ tgt)[None, :] + 1e-3 * z[::2]
    elif c.kind == "zero_rows":
        w["cb"][:, 1] = 0.0
        w["cb"][:, -1] = 0.0
    elif c.kind == "zero_e":   # codebook 1's in_proj makes e exactly 0
        w["in_w"][1] = 0.0
        w["in_b"][1] = 0.0
    z = model(z, c.dtype)
    if c.nan_frame >= 0:
        z[c.nan_frame, Z // 2] = float("nan")
    return dict(w=w, z=z)


def unit_rows(cb: torch.Tensor, dt) -> torch.Tensor:
    """F.normalize of the codebook as the model holds it, float64."""
    m = model(cb, dt)
    return m / m.norm(dim=-1, keepdim=True).clamp(min=1e-12)


def first_same(un: torch.Tensor) -> torch.Tensor:
    """[n_q, cs] -> the lowest index whose unit row is bit-identical to each row's."""
    out = torch.empty(un.shape[:2], dtype=torch.int64)
    for k in range(un.shape[0]):
        _, inv = torch.unique(un[k].cpu(), dim=0, return_inverse=True)
        first = torch.full((int(inv.max()) + 1,), un.shape[1], dtype=torch.int64)
        first.scatter_reduce_(0, inv, torch.arange(un.shape[1]), "amin")
        out[k] = first[inv]
    return out.to(un.device)


# ---- quantizer reference: check a launch's codes -----------------------------------------------------------------------------
def _cos(E: torch.Tensor, un: torch.Tensor) -> torch.Tensor:
    n = E.norm(dim=-1, keepdim=True)
    return (E / torch.where(n > 0, n, torch.ones_like(n))) @ un.T


def _box_points(lo_o: torch.Tensor, hi_o: torch.Tensor):
    """Every bf16 vector of a per-element box ([S, D] ord bounds, one per state): (state index, points [P, D] as ord)."""
    cnt = hi_o - lo_o + 1
    P = cnt.prod(dim=1)
    if int(P.max()) > CAP:
        raise AssertionError(f"{int(P.max())} points in one state's e box (cap {CAP})")
    fidx = torch.repeat_interleave(torch.arange(len(P), device=P.device), P)
    off = torch.cumsum(P, 0) - P
    local = torch.arange(len(fidx), device=P.device) - off[fidx]
    pts = torch.empty((len(fidx), lo_o.shape[1]), dtype=lo_o.dtype, device=lo_o.device)
    for d in range(lo_o.shape[1]):
        cd = cnt[fidx, d]
        pts[:, d] = lo_o[fidx, d] + local % cd
        local = local // cd
    return fidx, pts


FINE = 4          # an e element with more bf16 values than this in its box lies near 0: it is not enumerated (see the docstring)
SCAP = 32         # states per frame before they are merged into one interval state


def _sub(a: torch.Tensor, q: torch.Tensor) -> torch.Tensor:
    """rn(a - q) as the kernel computes it: fp32 subtraction of two bf16 values, then bf16."""
    return (a.float() - q.float()).bfloat16().double()


def _st(e: torch.Tensor, zq: torch.Tensor) -> torch.Tensor:
    """st = rn(e + rn(zq - e)), elementwise, exactly as fp32 then bf16 computes it."""
    return ((zq.float() - e.float()).bfloat16().float() + e.float()).bfloat16().double()


def _bf16_step(c, k, W, b, Wo, bo, un, fs, cbm, code, nanf, S, st):
    """One codebook of a bf16 launch over the set of states S: check the picks, then the states after the residual update."""
    dev, D, Z = code.device, c.D, c.Z
    F_ = code.shape[0]
    esim = (2 * D + 8) * U
    if len(S["f"]) == 0:   # no frame followed any more
        st["unfollowed"] += int((~nanf).sum())
        return torch.zeros(F_, dtype=torch.bool, device=dev), S
    sf, cS = S["f"], code[S["f"]]
    Wp, Wn = W.clamp(min=0), W.clamp(max=0)
    e64 = S["r"] @ W.T + b
    M = torch.maximum(S["lo"].abs(), S["hi"].abs()) @ W.abs().T
    Ee = (math.ceil(Z / 32) + 6) * U * M + U * (M + b.abs())
    lo_o = bf_ord(S["lo"] @ Wp.T + S["hi"] @ Wn.T + b - Ee)
    hi_o = bf_ord(S["hi"] @ Wp.T + S["lo"] @ Wn.T + b + Ee)
    near_o = bf_ord(e64)
    fine = hi_o - lo_o + 1 > FINE
    while True:   # a box still past CAP points: hold its widest enumerated element as well
        cnt = torch.where(fine, torch.ones_like(lo_o), hi_o - lo_o + 1)
        big = cnt.double().prod(dim=1) > CAP
        if not big.any():
            break
        fine[big, cnt[big].argmax(dim=1)] = True
    width = torch.where(fine, bf_from_ord(hi_o) - bf_from_ord(lo_o), torch.zeros_like(e64)).norm(dim=1)
    pidx, pts = _box_points(torch.where(fine, near_o, lo_o), torch.where(fine, near_o, hi_o))
    E = bf_from_ord(pts)
    pf = sf[pidx]
    st["points"] = max(st["points"], int(torch.bincount(pf).max()))
    cos = _cos(E, un)
    top = cos.topk(min(2, cos.shape[1]), dim=1).values
    best = top[:, 0]
    cp = cS[pidx]
    gap = best - cos.gather(1, cp[:, None])[:, 0]
    slack = 2 * esim + 4 * width[pidx] / E.norm(dim=1).clamp(min=1e-300)
    zero_e = (E == 0).all(dim=1) & ~fine[pidx].any(dim=1)
    ok = (gap <= slack) & (fs[cp] == cp) & (~zero_e | (cp == 0))
    near_pt = S["near"][pidx] & (pts == near_o[pidx]).all(dim=1)

    def per_frame(v):
        return torch.zeros(F_, dtype=torch.bool, device=dev).index_put_((pf,), v, accumulate=True)
    lost = S["lost"]
    valid = ~nanf & ~lost
    st["unfollowed"] += int((~nanf & lost).sum())
    any_ok = per_frame(ok)
    st["slack"] += int((any_ok & ~per_frame(ok & (gap <= 0)) & valid).sum())
    st["fine"] += int((any_ok & ~per_frame(ok & (gap <= 2 * esim)) & valid).sum())
    st["branch"] += int((any_ok & ~per_frame(ok & near_pt) & valid).sum())
    # a pick the check cannot tell from the runner-up: its slack reaches the gap between the two best similarities
    st["undecided"] += int((per_frame(ok & (best - top[:, -1] <= slack) & (cos.shape[1] > 1)) & valid).sum())
    g = torch.full((F_,), float("inf"), dtype=torch.float64, device=dev).scatter_reduce(
        0, pf, torch.where(ok, gap / (2 * esim), torch.full_like(gap, float("inf"))), "amin")[any_ok & valid]
    if g.numel():
        st["worst"] = max(st["worst"], float(g.max()))
    fail = ~any_ok & valid
    keep = ok | (~any_ok)[pf]          # a failed pick: continue from every point
    pidx, E, near_pt = pidx[keep], E[keep], near_pt[keep]
    zq = cbm[code[sf[pidx]]]
    stv = _st(E, zq)
    # a near-0 element was held at its nearest value: every other value of its range gives an st of its own (usually none)
    # (more than FINE distinct st values: the frame is no longer followed, and its later picks are counted as such)
    lost = lost.clone()
    for s_i, d in fine.nonzero().tolist():
        if lost[sf[s_i]] or int(hi_o[s_i, d] - lo_o[s_i, d]) > 1 << 16:
            lost[sf[s_i]] = True
            continue
        vals = torch.unique(_st(bf_from_ord(torch.arange(int(lo_o[s_i, d]), int(hi_o[s_i, d]) + 1, device=dev)).double(),
                                cbm[code[sf[s_i]], d]))
        if len(vals) > FINE:
            lost[sf[s_i]] = True
            continue
        rows = (pidx == s_i).nonzero()[:, 0]
        for v in vals.tolist():
            if rows.numel() and not (stv[rows, d] == v).all():
                extra = stv[rows].clone()
                extra[:, d] = v
                pidx, stv = torch.cat([pidx, pidx[rows]]), torch.cat([stv, extra])
                near_pt = torch.cat([near_pt, torch.zeros_like(rows, dtype=torch.bool)])
    alive = ~lost[sf[pidx]]
    pidx, stv, near_pt = pidx[alive], stv[alive], near_pt[alive]
    # the next states: one per (state, distinct st); the nearest path follows the nearest point where it was kept
    key, inv = torch.unique(torch.cat([pidx[:, None].double(), stv], dim=1), dim=0, return_inverse=True)
    par, stn = key[:, 0].long(), key[:, 1:]
    nf = torch.zeros(len(key), dtype=torch.bool, device=dev).index_put_((inv,), near_pt, accumulate=True)
    cf = sf[par]
    has = torch.zeros(F_, dtype=torch.bool, device=dev).index_put_((cf,), nf, accumulate=True)
    first = torch.ones(len(key), dtype=torch.bool, device=dev)
    first[1:] = cf[1:] != cf[:-1]
    nf = nf | (first & ~has[cf])
    q64 = stn @ Wo.T + bo
    Mq = stn.abs() @ Wo.abs().T
    Eq = (D + 1) * U * Mq + U * (Mq + bo.abs())
    N = dict(f=cf, r=_sub(S["r"][par], rn(q64)), lo=_sub(S["lo"][par], rn(q64 + Eq)), hi=_sub(S["hi"][par], rn(q64 - Eq)), near=nf)
    lost_f = lost
    cnt = torch.bincount(cf, minlength=F_)
    over = cnt > SCAP
    if over.any():   # too many paths in a frame: one state holding their union (sound, looser), counted
        st["merged"] += int(over.sum())
        lo = torch.full((F_, Z), float("inf"), dtype=torch.float64, device=dev).scatter_reduce(
            0, cf[:, None].expand(-1, Z), N["lo"], "amin")
        hi = torch.full((F_, Z), -float("inf"), dtype=torch.float64, device=dev).scatter_reduce(
            0, cf[:, None].expand(-1, Z), N["hi"], "amax")
        m = over[cf]
        keep_s = ~m | N["near"]
        N["lo"] = torch.where(m[:, None], lo[cf], N["lo"])
        N["hi"] = torch.where(m[:, None], hi[cf], N["hi"])
        N = {n: v[keep_s] for n, v in N.items()}
    if len(N["f"]):
        st["states"] = max(st["states"], int(torch.bincount(N["f"]).max()))
    N["lost"] = lost_f
    return fail, N


def check_codes(c: QCase, inp: dict, codes: torch.Tensor) -> dict:
    """Follow the launch's codes [F, n_q] through the reference; count the picks that fail and the near ties."""
    w, z, dt = inp["w"], inp["z"], c.dtype
    dev = z.device
    F_, D, Z = z.shape[0], c.D, c.Z
    un = unit_rows(w["cb"], dt)
    fs = first_same(un)
    cbm = model(w["cb"], dt)
    esim = (2 * D + 8) * U
    nanf = torch.isnan(z).any(dim=1)
    r = torch.where(nanf[:, None], torch.zeros_like(z), z)
    d_r = torch.zeros_like(r)
    # bf16: the kernel's possible paths, one row each: frame, nearest residual, residual interval, on the nearest path
    states = dict(f=torch.arange(F_, device=dev), r=r, lo=r.clone(), hi=r.clone(), near=torch.ones(F_, dtype=torch.bool, device=dev),
                  lost=torch.zeros(F_, dtype=torch.bool, device=dev))
    st = dict(picks=0, fail=0, slack=0, branch=0, fine=0, undecided=0, merged=0, unfollowed=0, points=1, states=1, worst=0.0,
              fail_at=None)
    for k in range(c.n_q):
        W, b = model(w["in_w"][k], dt), model(w["in_b"][k], dt)
        Wo, bo = model(w["out_w"][k], dt), model(w["out_b"][k], dt)
        code = codes[:, k].to(dev)
        st["picks"] += int((~nanf).sum())
        bad_nan = nanf & (code != 0)
        M = (r.abs() + d_r) @ W.abs().T
        e64 = r @ W.T + b
        Ee = (math.ceil(Z / 32) + 6) * U * M + U * (M + b.abs())
        if dt == BF:
            fail, states = _bf16_step(c, k, W, b, Wo, bo, un[k], fs[k], cbm[k], code, nanf, states, st)
            fail = fail | bad_nan
        else:
            Ee = Ee + d_r @ W.abs().T
            cos = _cos(e64, un[k])
            best = cos.max(dim=1).values
            ck = cos.gather(1, code[:, None])[:, 0]
            en = e64.norm(dim=1)
            slack = 2 * esim + 4 * Ee.norm(dim=1) / en.clamp(min=1e-300)
            zero_e = (e64 == 0).all(dim=1) & (Ee == 0).all(dim=1)
            gap = best - ck
            st["undecided"] += int((((best - cos.topk(min(2, cos.shape[1]), dim=1).values[:, -1]) <= slack)
                                    & (cos.shape[1] > 1) & ~nanf).sum())
            ok = ((gap <= slack) | (en <= Ee.norm(dim=1))) & (fs[k][code] == code) & (~zero_e | (code == 0))
            valid = ~nanf
            st["slack"] += int((ok & (gap > 0) & valid).sum())
            g = (gap / slack)[ok & valid & (en > Ee.norm(dim=1))]
            if g.numel():
                st["worst"] = max(st["worst"], float(g.max()))
            fail = (~ok & valid) | bad_nan
            zq = cbm[k][code]
            d_st = 3 * U * (zq.abs() + e64.abs() + Ee)
            q = zq @ Wo.T + bo
            Mq = zq.abs() @ Wo.abs().T
            d_q = (D + 1) * U * Mq + d_st @ Wo.abs().T + U * (q.abs() + Mq + bo.abs())
            r = r - q
            d_r = d_r + d_q + U * r.abs()
        nf = int(fail.sum())
        if nf and st["fail_at"] is None:
            f = int(fail.nonzero()[0])
            st["fail_at"] = (f, k, int(code[f]))
        st["fail"] += nf
    return st


# ---- a simulated kernel (nearest roundings), and its modelled bugs -------------------------------------------------------------
Q_BUGS = ("st_unrounded", "res_unrounded", "in_bias_other", "in_bias_missing", "out_bias_other", "out_bias_missing",
          "rows_unnormalised", "rows_unrounded", "ties_high")


def simulate(c: QCase, inp: dict, bug: str | None = None) -> torch.Tensor:
    """The kernel's arithmetic in float64 with every fp32 sum exact and every rounding to bf16 to nearest: codes [F, n_q]."""
    w, z, dt = inp["w"], inp["z"], c.dtype
    bf = dt == BF
    r = z.clone()
    nanf = torch.isnan(z).any(dim=1)
    un = unit_rows(w["cb"], F32 if bug == "rows_unrounded" else dt)
    if bug == "rows_unnormalised":
        un = model(w["cb"], dt)
    cbm = model(w["cb"], dt)
    n_q = c.n_q
    out = []
    for k in range(n_q):
        W, b = model(w["in_w"][k], dt), model(w["in_b"][k], dt)
        Wo, bo = model(w["out_w"][k], dt), model(w["out_b"][k], dt)
        if bug == "in_bias_other":
            b = model(w["in_b"][(k + 1) % n_q], dt)
        if bug == "in_bias_missing":
            b = torch.zeros_like(b)
        if bug == "out_bias_other":
            bo = model(w["out_b"][(k + 1) % n_q], dt)
        if bug == "out_bias_missing":
            bo = torch.zeros_like(bo)
        e = model(r @ W.T + b, dt)
        cos = _cos(e, un[k])
        if bug == "ties_high":
            code = cos.shape[1] - 1 - cos.flip(1).argmax(dim=1)
        elif bug == "runner_up_last" and k == n_q - 1:
            code = cos.topk(2, dim=1).indices[:, 1]
        else:
            code = cos.argmax(dim=1)
        code = torch.where(nanf | (e == 0).all(dim=1), torch.zeros_like(code), code)
        zq = cbm[k][code]
        if bf and bug != "st_unrounded":
            stv = ((zq.float() - e.float()).bfloat16().float() + e.float()).bfloat16().double()
        else:
            stv = e + (zq - e)
        q = model(stv @ Wo.T + bo, dt)
        r = (r.float() - q.float()).bfloat16().double() if (bf and bug != "res_unrounded") else r - q
        out.append(code)
    return torch.stack(out, dim=1)


# ---- from_codes cases and reference -------------------------------------------------------------------------------------------
@dataclasses.dataclass
class FCase:
    dtype: torch.dtype
    K: int
    D: int
    C: int
    B: int = 2
    T: int = 5
    cs: int = 37
    ragged: bool = False
    window: tuple | None = None  # (m_lo, m_hi)
    seed: int = 0

    @property
    def id(self):
        s = f"{dtn(self.dtype)}-K{self.K}-D{self.D}-C{self.C}-B{self.B}T{self.T}"
        if self.ragged:
            s += "-ragged"
        if self.window is not None:
            s += f"-window{self.window[0]}_{self.window[1]}"
        return s

    @property
    def codes_T(self):
        return self.T + 6 if self.window is not None else self.T


F_SHAPES = [(1, 1), (3, 5), (9, 8), (16, 16), (32, 8)]
F_WIDTHS = [1, 64, 255, 256, 257, 1024, 1536]
F_CASES = [FCase(dt, K, D, C) for dt in (BF, F32) for (K, D) in F_SHAPES for C in F_WIDTHS]
F_RAGGED = [FCase(dt, 9, 8, 257, B=6, T=7, ragged=True) for dt in (BF, F32)] + [FCase(BF, 32, 8, 64, B=6, T=4, ragged=True)]
F_WINDOW = [FCase(dt, 9, 8, 96, B=8, T=12, window=m) for dt in (BF, F32) for m in ((0, 0), (10, 10))] + \
           [FCase(BF, 3, 5, 1, B=8, T=1, window=(0, 0))]


def make_f(c: FCase) -> dict:
    g = torch.Generator().manual_seed(500 + c.seed + c.K * 13 + c.D * 7 + c.C)
    w = dict(cb=torch.randn(c.K, c.cs, c.D, generator=g).double(),
             w=(torch.randn(c.K, c.C, c.D, generator=g) / math.sqrt(c.D)).double(),
             b=(torch.randn(c.K, c.C, generator=g) * 0.1).double())
    n_valid = c.cs - 1 if (c.ragged or c.window is not None) else c.cs
    codes = torch.randint(0, n_valid, (c.B, c.K, c.codes_T), generator=g)
    codes[0, :, 0] = 0
    codes[-1, :, -1] = n_valid - 1
    d = dict(w=w, codes=codes)
    if c.ragged or c.window is not None:
        w["cb"][:, -1] = float("nan")     # the row every code that must not be read points at
        fl = [-1, 0, 1, c.T - 1, c.T, c.T + 5] + [c.T // 2] * c.B
        d["lengths"] = torch.tensor(fl[:c.B], dtype=torch.int32)
    if c.window is not None:
        n = d["lengths"].clamp(0, c.T)
        cT = c.codes_T
        starts = [-3, 0, 2, cT, cT - int(n[4]) + 4, 1, 3, -1][:c.B]
        lo = [0, 1, -2, 2, 0, 3, 5, 1][:c.B]
        hi = [3, 1, 100, 1, c.T, 2, 4, 2][:c.B]          # normal, empty, clamped, reversed, ...
        d["start"] = torch.tensor(starts, dtype=torch.int32)
        d["emit_lo"], d["emit_hi"] = torch.tensor(lo, dtype=torch.int32), torch.tensor(hi, dtype=torch.int32)
        for b in range(c.B):   # codes outside each row's window point at the NaN row
            s = min(max(starts[b], 0), cT - int(n[b]))
            keep = torch.zeros(cT, dtype=torch.bool)
            keep[s:s + int(n[b])] = True
            codes[b][:, ~keep] = c.cs - 1
    elif c.ragged:
        n = d["lengths"].clamp(0, c.T)
        for b in range(c.B):
            codes[b, :, int(n[b]):] = c.cs - 1
    return d


def from_codes_ref(c: FCase, w: dict, codes: torch.Tensor, bug: str | None = None) -> dict:
    """codes [R, K] (one code frame per row) -> nearest value, candidate interval (bf16) or bar (f32), each [R, C]."""
    dt = c.dtype
    cb, W, bvec = model(w["cb"], dt), model(w["w"], dt), model(w["b"], dt)
    R = codes.shape[0]
    acc = lo = hi = None
    err = torch.zeros(R, c.C, dtype=torch.float64, device=codes.device)
    for k in range(c.K):
        e = cb[k][codes[:, k]]                                  # [R, D]
        s64 = e @ W[k].T + bvec[k]
        Es = (c.D + 1) * U * (e.abs() @ W[k].abs().T) + U * s64.abs()
        if dt == BF:
            s, s_lo, s_hi = rn(s64), rn(s64 - Es), rn(s64 + Es)
            if k == 0:
                acc, lo, hi = s, s_lo, s_hi
            elif bug == "sum_fp32":
                acc, lo, hi = acc + s, lo + s_lo, hi + s_hi
            else:
                def add(a, x):
                    return (a.float() + x.float()).bfloat16().double()
                acc, lo, hi = add(acc, s), add(lo, s_lo), add(hi, s_hi)
        else:
            acc = s64 if k == 0 else acc + s64
            err = err + Es + (U * acc.abs() if k else 0)
    if dt == BF:
        if bug == "sum_fp32":
            acc = rn(acc)
        return dict(ref=acc, lo=lo, hi=hi)
    return dict(ref=acc, bar=err + 1e-300)


def expected_frames(c: FCase, d: dict, bug: str | None = None):
    """Per latent frame (b, t): the code frame it reads (-1: a zero latent, -2: left as it is)."""
    src = torch.full((c.B, c.T), 0, dtype=torch.int64)
    for b in range(c.B):
        n = c.T if "lengths" not in d else min(max(int(d["lengths"][b]), 0), c.T)
        need = (0, c.T)
        s = 0
        if c.window is not None:
            lo = min(max(int(d["emit_lo"][b]), 0), n)
            hi = min(max(int(d["emit_hi"][b]), lo), n)
            need = (0, 0) if lo == hi else (lo - c.window[0], hi + c.window[1])
            s = 0 if bug == "window_no_offset" else min(max(int(d["start"][b]), 0), c.codes_T - n)
        for t in range(c.T):
            if not (need[0] <= t < need[1]):
                src[b, t] = -2
            elif t >= n and bug != "ragged_tail_computed":
                src[b, t] = -1
            else:
                src[b, t] = s + t
    return src


def check_from_codes(c: FCase, d: dict, got: torch.Tensor, bug: str | None = None) -> tuple:
    """got [B, T, C] (float64, NaN where unwritten): (values outside their candidate set or past the bar, worst f32 error /
    bar, two-candidate values)."""
    src = expected_frames(c, d, bug)
    dev = got.device
    codes = d["codes"].to(dev)
    bad = 0
    worst, two = 0.0, 0
    left = src == -2
    zero = src == -1
    left_d, zero_d = left.to(dev), zero.to(dev)
    bad += int((~torch.isnan(got[left_d])).sum())
    bad += int((got[zero_d] != 0).sum())
    live = (src >= 0).to(dev)
    if live.any():
        bi, ti = live.nonzero(as_tuple=True)
        cf = codes[bi, :, src.to(dev)[bi, ti].clamp(min=0, max=c.codes_T - 1)]   # [R, K]
        ref = from_codes_ref(c, {k: v.to(dev) for k, v in d["w"].items()}, cf, bug if bug == "sum_fp32" else None)
        g = got[bi, ti]
        if c.dtype == BF:
            o = bf_ord(g)
            ok = (o >= bf_ord(ref["lo"])) & (o <= bf_ord(ref["hi"])) & ~torch.isnan(g)
            bad += int((~ok).sum())
            two = int((bf_ord(ref["hi"]) > bf_ord(ref["lo"])).sum())
        else:
            r = (g - ref["ref"]).abs() / ref["bar"]
            r = torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)
            worst = float(r.max())
            bad += int((r > 1).sum())
    return bad, worst, two


# ---- running the hooks -----------------------------------------------------------------------------------------------------
def q_scratch_bytes(c: QCase) -> int:
    return 4 * c.n_q * c.cs * c.D + 4 * c.n_q * (2 * c.D * c.Z + c.D + c.cs * c.D + c.Z) + 6 * 256


def run_quantize(c: QCase, w: dict, z: torch.Tensor, lengths=None, hop=0, pad=5):
    """One launch: (codes [F, n_q], z after [F, Z] float64, unit rows from scratch, tails of both buffers)."""
    from parler_tts_b200 import _lib
    dt = c.dtype
    src = {k: v.float().to(DEV).contiguous() for k, v in w.items()}
    F_ = c.B * c.T
    zb = torch.full((F_ + pad, c.Z), float("nan"), dtype=dt, device=DEV)
    zb[:F_] = z.to(dt).to(DEV)
    codes = torch.full((c.B * c.n_q * c.T + pad,), -7, dtype=torch.int64, device=DEV)
    scratch = torch.empty(q_scratch_bytes(c), dtype=torch.uint8, device=DEV)
    sl = None if lengths is None else torch.tensor(lengths, dtype=torch.int32, device=DEV)
    _lib.check(_lib.lib().ptts_op_dac_quantize(
        _lib.dtype_code(dt), _lib.F32, c.B, c.T, c.Z, c.D, c.n_q, c.cs, _lib.ptr(src["in_w"]), _lib.ptr(src["in_b"]),
        _lib.ptr(src["cb"]), _lib.ptr(src["out_w"]), _lib.ptr(src["out_b"]), _lib.ptr(zb), _lib.ptr(sl), hop,
        _lib.ptr(codes), _lib.ptr(scratch), _lib.stream_ptr()))
    torch.cuda.synchronize()
    cf = codes[:-pad].view(c.B, c.n_q, c.T).permute(0, 2, 1).reshape(F_, c.n_q)
    rows = scratch[:4 * c.n_q * c.cs * c.D].view(torch.float32).view(c.n_q, c.cs, c.D).double()
    return cf, zb[:F_].double(), rows, codes[-pad:], zb[F_:]


def _q_stats(c, st):
    s = QSTATS.setdefault(dtn(c.dtype), dict(cases=0))
    s["cases"] += 1
    for key in ("picks", "slack", "fine", "branch", "undecided", "merged", "unfollowed"):
        s[key] = s.get(key, 0) + st[key]
    for key in ("points", "states", "worst"):
        s[key] = max(s.get(key, 0), st[key])


def check_quantize_case(c: QCase):
    inp = make_q(c)
    inp_d = dict(w={k: v.to(DEV) for k, v in inp["w"].items()}, z=inp["z"].to(DEV))
    codes, z_after, rows, ctail, ztail = run_quantize(c, inp["w"], inp["z"])
    codes2, _, _, _, _ = run_quantize(c, inp["w"], inp["z"])
    assert torch.equal(codes, codes2), f"{c.id}: two launches differ"
    assert (ctail == -7).all() and torch.isnan(ztail.float()).all(), f"{c.id}: written past B * T"
    assert ((codes >= 0) & (codes < c.cs)).all(), f"{c.id}: a code outside [0, cs) or a frame not written"
    zin = inp_d["z"]
    assert torch.equal(torch.isnan(z_after), torch.isnan(zin)) and torch.equal(z_after.nan_to_num(), zin.nan_to_num()), \
        f"{c.id}: the latents changed"
    # the packed unit rows
    ref_rows = unit_rows(inp_d["w"]["cb"], c.dtype)
    bar = (c.D / 2 + 3) * U * ref_rows.abs()
    err = (rows - ref_rows).abs()
    assert (err <= bar).all(), f"{c.id}: unit row off by {float((err / bar.clamp(min=1e-300)).max()):.2f}x its bound"
    st = check_codes(c, inp_d, codes)
    _q_stats(c, st)
    assert st["fail"] == 0, f"{c.id}: {st['fail']} picks outside the reference, first (frame, codebook, code) {st['fail_at']}"
    if c.nan_frame >= 0:
        assert (codes[c.nan_frame] == 0).all(), f"{c.id}: the NaN frame did not code 0"
        z2 = inp["z"].clone()
        z2[c.nan_frame] = 0.0
        other, _, _, _, _ = run_quantize(c, inp["w"], z2)
        keep = torch.arange(c.B * c.T, device=DEV) != c.nan_frame
        assert torch.equal(codes[keep], other[keep]), f"{c.id}: the NaN frame moved its neighbours' codes"
    return codes


# ---- GPU tests -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    for dt, s in sorted(QSTATS.items()):
        print(f"\n[dac quantizer reference] quantize {dt}: {s['cases']} cases, {s['picks']} picks, {s['slack']} needed slack, "
              f"{s['fine']} more than 2 E_sim, {s['branch']} an ambiguous-rounding branch, {s['undecided']} undecided, "
              f"{s['merged']} merged frames, {s['unfollowed']} not followed, at most {s['points']} e points and {s['states']} states per frame, "
              f"worst gap / bar {s['worst']:.3f}")
    for dt, (n, vals, two, worst) in sorted(FSTATS.items()):
        print(f"\n[dac quantizer reference] from_codes {dt}: {n} cases, {vals} values"
              + (f", {two} with two or more candidates" if dt == "bf16" else f", worst error / bar {worst:.3f}"))


@pytest.mark.gpu
@pytest.mark.parametrize("c", Q_CASES, ids=lambda c: c.id)
def test_quantize(c):
    check_quantize_case(c)


@pytest.mark.gpu
def test_quantize_real_shape():
    """The 44.1 kHz codec's quantizer (latent 1024, 9 codebooks of 1024 x 8) over 32 clips of 173 frames."""
    check_quantize_case(Q_REAL)


@pytest.mark.gpu
@pytest.mark.parametrize("c", Q_RAGGED, ids=lambda c: c.id)
def test_quantize_ragged(c):
    inp = make_q(c)
    hop, samples = c.ragged, c.T * c.ragged
    lengths = [-1, 0, 1, hop - 1, hop, hop + 1, samples, samples + 7][:c.B]
    full, _, _, _, _ = run_quantize(c, inp["w"], inp["z"])
    codes, z_after, _, ctail, ztail = run_quantize(c, inp["w"], inp["z"], lengths, hop)
    assert (ctail == -7).all() and torch.isnan(ztail.float()).all(), f"{c.id}: written past B * T"
    zin = inp["z"].to(DEV)
    for b, n in enumerate(lengths):
        Fb = -(-min(max(n, 1), samples) // hop)
        fr = slice(b * c.T, (b + 1) * c.T)
        cb_, zb_ = codes[fr], z_after[fr]
        assert (cb_[Fb:] == c.cs).all(), f"{c.id}: row {b} (length {n}) frames past {Fb} do not hold codebook_size"
        assert (zb_[Fb:] == 0).all(), f"{c.id}: row {b} frames past {Fb} are not zero latents"
        assert torch.equal(cb_[:Fb], full[fr][:Fb]), f"{c.id}: row {b} codes differ from the non-ragged launch"
        assert torch.equal(zb_[:Fb], zin[fr][:Fb]), f"{c.id}: row {b} latents changed"


def run_from_codes(c: FCase, d: dict, pad=3):
    from parler_tts_b200 import _lib
    dt = c.dtype
    w = {k: v.float().to(DEV).contiguous() for k, v in d["w"].items()}
    codes = d["codes"].to(DEV).contiguous()
    z = torch.full((c.B * c.T + pad, c.C), float("nan"), dtype=dt, device=DEV)
    scratch = torch.empty((c.K * (c.cs + c.C) * c.D + c.K * c.C) * 4 + 3 * 256, dtype=torch.uint8, device=DEV)
    dv = {k: d[k].to(DEV) if k in d else None for k in ("lengths", "start", "emit_lo", "emit_hi")}
    m_lo, m_hi = c.window if c.window is not None else (0, 0)
    _lib.check(_lib.lib().ptts_op_dac_from_codes(
        _lib.dtype_code(dt), _lib.F32, c.B, c.K, c.D, c.C, c.T, c.cs, _lib.ptr(codes), c.codes_T, _lib.ptr(w["cb"]),
        _lib.ptr(w["w"]), _lib.ptr(w["b"]), _lib.ptr(dv["lengths"]), _lib.ptr(dv["start"]), _lib.ptr(dv["emit_lo"]),
        _lib.ptr(dv["emit_hi"]), m_lo, m_hi, _lib.ptr(z), _lib.ptr(scratch), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return z[:c.B * c.T].view(c.B, c.T, c.C).double(), z[c.B * c.T:]


def check_from_codes_case(c: FCase):
    d = make_f(c)
    got, tail = run_from_codes(c, d)
    got2, _ = run_from_codes(c, d)
    assert torch.isnan(tail.float()).all(), f"{c.id}: written past B * T"
    assert torch.equal(got.nan_to_num(nan=7.0), got2.nan_to_num(nan=7.0)), f"{c.id}: two launches differ"
    bad, worst, two = check_from_codes(c, d, got)
    s = FSTATS.setdefault(dtn(c.dtype), [0, 0, 0, 0.0])
    s[0] += 1
    s[1] += int((~torch.isnan(got)).sum())
    s[2] += two
    s[3] = max(s[3], worst)
    assert bad == 0, f"{c.id}: {bad} values outside the reference (worst f32 error / bar {worst:.2f})"


@pytest.mark.gpu
@pytest.mark.parametrize("c", F_CASES, ids=lambda c: c.id)
def test_from_codes(c):
    check_from_codes_case(c)


@pytest.mark.gpu
@pytest.mark.parametrize("c", F_RAGGED + F_WINDOW, ids=lambda c: c.id)
def test_from_codes_ragged_and_windowed(c):
    check_from_codes_case(c)


@pytest.mark.gpu
def test_refusals():
    """PTTS_EINVAL with nothing written for the shapes the launchers refuse."""
    from parler_tts_b200 import _lib
    buf = torch.zeros(1 << 16, dtype=torch.float32, device=DEV)
    codes = torch.full((1 << 12,), -7, dtype=torch.int64, device=DEV)
    z = torch.full((1 << 14,), float("nan"), dtype=torch.float32, device=DEV)
    scratch = torch.full((1 << 18,), 0xAB, dtype=torch.uint8, device=DEV)
    fl = torch.tensor([2, 2], dtype=torch.int32, device=DEV)
    p = _lib.ptr(buf)

    def quant(D=8, Z=64, sl=None, hop=0, dtype=_lib.F32):
        return _lib.check(_lib.lib().ptts_op_dac_quantize(dtype, _lib.F32, 2, 3, Z, D, 2, 16, p, p, p, p, p, _lib.ptr(z), sl, hop,
                                                          _lib.ptr(codes), _lib.ptr(scratch), _lib.stream_ptr()))

    def fc(K=4, D=8, T=3, codes_T=3, lengths=None, start=None, window=False, dtype=_lib.F32):
        e = _lib.ptr(fl) if window else None
        return _lib.check(_lib.lib().ptts_op_dac_from_codes(dtype, _lib.F32, 2, K, D, 16, T, 4, _lib.ptr(codes), codes_T, p, p, p,
                                                            lengths, start, e, e, 0, 0, _lib.ptr(z), _lib.ptr(scratch),
                                                            _lib.stream_ptr()))
    refused = [lambda: quant(D=2), lambda: quant(D=12), lambda: quant(D=32), lambda: quant(Z=0), lambda: quant(Z=1537),
               lambda: quant(sl=_lib.ptr(fl), hop=0), lambda: quant(dtype=2),
               lambda: fc(K=33, D=1), lambda: fc(D=17), lambda: fc(K=17, D=16), lambda: fc(window=True, start=_lib.ptr(fl)),
               lambda: fc(window=True, lengths=_lib.ptr(fl)), lambda: fc(window=True, lengths=_lib.ptr(fl), start=_lib.ptr(fl),
                                                                          T=4, codes_T=3),
               lambda: fc(codes_T=4), lambda: fc(dtype=2)]
    for call in refused:
        with pytest.raises(ValueError):
            call()
    torch.cuda.synchronize()
    assert (codes == -7).all() and torch.isnan(z).all() and (scratch == 0xAB).all(), "a refused call wrote something"


# ---- host tests ------------------------------------------------------------------------------------------------------------
def test_hooks_are_bound():
    from parler_tts_b200 import _lib
    assert len(_lib._SIGS["ptts_op_dac_quantize"][1]) == 19
    assert len(_lib._SIGS["ptts_op_dac_from_codes"][1]) == 22


def _golden_inputs():
    from tests.golden.make_dac_encode_golden import encode_cfg, weights
    cfg = encode_cfg()
    w = weights(cfg)
    n_q = cfg.n_codebooks
    q = "quantizer.quantizers.{}."
    st = lambda key, f=lambda t: t: torch.stack([f(w[q.format(i) + key]) for i in range(n_q)]).double()   # noqa: E731
    ww = dict(in_w=st("in_proj.weight", lambda t: t[:, :, 0]), in_b=st("in_proj.bias"), cb=st("codebook.weight"),
              out_w=st("out_proj.weight", lambda t: t[:, :, 0]), out_b=st("out_proj.bias"))
    return cfg, w, ww


def test_quantize_reference_reproduces_oracle(golden_dir):
    """With every rounding off, the simulated kernel is OracleDACEncoder.quantize in float64, and both give the fixture's codes
    wherever the fixture's margin (best - second similarity) is clear of fp32 noise."""
    from tests.dac_encode_oracle import OracleDACEncoder
    cfg, w, ww = _golden_inputs()
    g = np.load(os.path.join(golden_dir, "dac_encode.npz"))
    lat = torch.from_numpy(g["latents"])                        # [B, Z, T]
    B, Z, T = lat.shape
    o = OracleDACEncoder(cfg, w, torch.float64)
    ocodes, _ = o.quantize(lat)
    c = QCase(torch.float64, cfg.codebook_dim, Z, cfg.codebook_size, cfg.n_codebooks, B, T)
    z = lat.permute(0, 2, 1).reshape(B * T, Z)
    sim = simulate(c, dict(w=ww, z=z))
    assert torch.equal(sim, ocodes.permute(0, 2, 1).reshape(B * T, -1))
    clear = torch.from_numpy(g["margins"]).permute(1, 2, 0).reshape(B * T, -1) > 1e-4
    assert clear.float().mean() > 0.9
    fix = torch.from_numpy(g["codes"]).permute(0, 2, 1).reshape(B * T, -1)
    assert torch.equal(sim[clear], fix[clear])
    st = check_codes(c, dict(w=ww, z=z), ocodes.permute(0, 2, 1).reshape(B * T, -1))   # the checker itself, in float64
    assert st["fail"] == 0 and st["picks"] == B * T * cfg.n_codebooks, st
    wrong = fix.clone()
    wrong[:, -1] = (wrong[:, -1] + 1) % cfg.codebook_size
    assert check_codes(c, dict(w=ww, z=z), wrong)["fail"] >= B * T * 0.9


def test_from_codes_reference_matches_oracle():
    """The from_codes reference is OracleDAC.from_codes: in float64 (f32 reference value) and in bf16 (member of the set)."""
    from oracle.dac import OracleDAC
    cfg, w, ww = _golden_inputs()
    K = cfg.n_codebooks
    c = FCase(F32, K, cfg.codebook_dim, cfg.hidden_size, B=2, T=6, cs=cfg.codebook_size)
    codes = torch.randint(0, c.cs, (2, K, 6), generator=torch.Generator().manual_seed(3))
    fw = dict(cb=ww["cb"], w=ww["out_w"], b=ww["out_b"])
    rows = codes.permute(0, 2, 1).reshape(-1, K)
    for dt in (F32, BF):
        ref = from_codes_ref(dataclasses.replace(c, dtype=dt), fw, rows)
        if dt == F32:
            got = OracleDAC(cfg, w, torch.float64).from_codes(codes).permute(0, 2, 1).reshape(-1, c.C)
            assert ((got - ref["ref"]).abs() <= ref["bar"]).all()
        else:
            got = OracleDAC(cfg, w, torch.bfloat16).from_codes(codes).permute(0, 2, 1).reshape(-1, c.C).double()
            o = bf_ord(got)
            assert ((o >= bf_ord(ref["lo"])) & (o <= bf_ord(ref["hi"]))).all()
            assert torch.equal(got, ref["ref"])


SIM_CASES = [QCase(BF, 4, 64, 4096, 4, 40, 20, seed=2), QCase(BF, 8, 64, 1024, 4, 2, 16, kind="dup"),
             QCase(BF, 16, 32, 2, 3, 1, 16, kind="zero_rows"), QCase(BF, 8, 33, 31, 3, 1, 9, kind="zero_e"),
             QCase(F32, 4, 64, 4096, 4, 40, 20, seed=2), QCase(F32, 8, 64, 1024, 4, 2, 16, kind="dup")]


@pytest.mark.parametrize("c", SIM_CASES, ids=lambda c: c.id)
def test_simulated_kernel_passes(c):
    """A kernel with every fp32 sum exact and every rounding to nearest is inside the reference on every pick."""
    inp = make_q(c)
    st = check_codes(c, inp, simulate(c, inp))
    assert st["fail"] == 0, st


def _bug_case(bug, dt=BF):
    if bug == "ties_high":
        return QCase(dt, 8, 64, 1024, 4, 2, 16, kind="dup")
    return QCase(dt, 4, 64, 4096, 4, 40, 20, seed=2)


Q_SENS = [(b, BF) for b in Q_BUGS] + \
         [(b, F32) for b in ("in_bias_other", "in_bias_missing", "out_bias_other", "out_bias_missing", "rows_unnormalised",
                             "ties_high")]


@pytest.mark.parametrize("bug,dt", Q_SENS, ids=[f"{b}-{dtn(d)}" for b, d in Q_SENS])
def test_quantize_sensitivity(bug, dt):
    """Each modelled quantizer bug fails two or more picks of its case."""
    c = _bug_case(bug, dt)
    inp = make_q(c)
    if bug == "rows_unrounded":   # fp32 codebook values a bf16 model rounds
        assert not torch.equal(rn(inp["w"]["cb"]), inp["w"]["cb"])
    st = check_codes(c, inp, simulate(c, inp, bug))
    assert st["fail"] >= 2, f"{bug} fails only {st['fail']} picks of {c.id}"


F_SENS = [("sum_fp32", FCase(BF, 9, 8, 257)), ("sum_fp32", FCase(BF, 32, 8, 64)),
          ("window_no_offset", FCase(BF, 9, 8, 96, B=8, T=12, window=(0, 0))),
          ("window_no_offset", FCase(F32, 9, 8, 96, B=8, T=12, window=(10, 10))),
          ("ragged_tail_computed", FCase(BF, 9, 8, 257, B=6, T=7, ragged=True)),
          ("ragged_tail_computed", FCase(F32, 9, 8, 96, B=8, T=12, window=(10, 10)))]


@pytest.mark.parametrize("bug,c", F_SENS, ids=[f"{b}-{c.id}" for b, c in F_SENS])
def test_from_codes_sensitivity(bug, c):
    """Each modelled from_codes bug puts two or more values outside their candidate sets (bf16) or past 4x the bar (f32)."""
    d = make_f(c)
    good = _simulate_from_codes(c, d)
    assert check_from_codes(c, d, good)[0] == 0
    bad = _simulate_from_codes(c, d, bug)
    n, worst, _ = check_from_codes(c, d, bad)
    if c.dtype == F32 and bug not in ("window_no_offset", "ragged_tail_computed"):
        assert worst > 4.0
    else:
        assert n >= 2, f"{bug}: only {n} values outside the reference"


def _simulate_from_codes(c: FCase, d: dict, bug: str | None = None) -> torch.Tensor:
    """The kernel's output with exact fp32 sums, nearest roundings and the modelled bug: [B, T, C], NaN where not written."""
    src = expected_frames(c, d, bug if bug in ("window_no_offset", "ragged_tail_computed") else None)
    out = torch.full((c.B, c.T, c.C), float("nan"), dtype=torch.float64)
    for b in range(c.B):
        for t in range(c.T):
            f = int(src[b, t])
            if f == -1:
                out[b, t] = 0.0
            elif f >= 0:
                cf = d["codes"][b, :, f][None]
                r = from_codes_ref(c, d["w"], cf, bug if bug == "sum_fp32" else None)
                out[b, t] = r["ref"][0]
    return out


def test_runner_up_caught_at_the_real_shape():
    """At the 44.1 kHz codec's quantizer shape (2 x 173 frames), a kernel that takes the runner-up at the last codebook fails the
    bf16 check in nearly every frame: the states keep the check tight through every codebook."""
    c = dataclasses.replace(Q_REAL, B=2)
    inp = make_q(c)
    good = simulate(c, inp)
    st = check_codes(c, inp, good)
    assert st["fail"] == 0 and st["undecided"] <= 0.02 * st["picks"], st
    bad = simulate(c, inp, "runner_up_last")
    assert torch.equal(bad[:, :-1], good[:, :-1])
    n = check_codes(c, inp, bad)["fail"]
    assert n >= 0.9 * c.B * c.T, f"the runner-up at the last codebook fails only {n} of {c.B * c.T} frames"
