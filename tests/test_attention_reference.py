"""The attention sweeps on their own, against a float64 reference, through the ptts_op_attention hook.

Sweeps: attention_decode_kernel (q_len == 1: two warps per (row, K/V head) item, 32-key bf16 / 16-key fp32 chunks taken
alternately), attention_prefill_tc_kernel (bf16 MHA prefill, tensor cores, 32-key chunks) and attention_kernel /
attention_item (fp32 or GQA prefill, or any prefill with prefill_sweep = 1).

The reference sees exactly the values the kernel sees: the query after the model-dtype rotary embedding, the cache rows and
the mask as an exclusion of keys; it computes softmax(q K^T / 8) V in float64.  Bars:
  bf16: |got - ref| <= 2^-8 (|ref| + sum_i p_i |v_i|) + 1e-6 -- the probabilities are rounded to bf16 before P V (relative
        error 2^-9 on each term of the numerator, sum_i p_i |v_i| in all) and so is the output (2^-9 |out|);
  fp32: |got - ref| <= 1e-5 sum_i p_i |v_i|.
Random keys make attention nearly uniform and hide errors, so every case plants structure (needles, masked needles, rising /
falling / widely spread scores, a rotary decoy) and its host test checks that the reference under a plausible kernel bug
(needle dropped, mask ignored, rotary position off by one, own key omitted, partial last chunk dropped, running maximum not
rescaled, first chunk dropped) moves by more than 4x the bar: a case that cannot see those bugs is not doing its job.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import math

import numpy as np
import pytest
import torch

HD = 64
MAX_POS = 4096       # rotary table rows the kernels may read: positions up to 4095 (max_position_embeddings - 1)
GAP = 40.0           # score of a needle above the rest

DECODE_N = [1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 95, 96, 97, 1023, 1024, 1025, 2047, 2048, 2049, 2579, 4095]
PREFILL_Q = [2, 9, 33, 65, 257, 2049]
CROSS_S = [1, 7, 31, 32, 33, 64, 200, 512]
BATCHES = (5, 1, 32)


# ---- the cache layout -------------------------------------------------------------------------------------------------
def kv_swz(t, d):
    """Position of element d of cached row t inside its 64-wide row (common.cuh): the 8-element chunk index XOR t % 8."""
    return ((((d >> 3) ^ t) & 7) << 3) | (d & 7)


def _swz_index(T: int) -> torch.Tensor:
    return kv_swz(torch.arange(T)[:, None], torch.arange(HD)[None, :])


def swizzle(rows: torch.Tensor) -> torch.Tensor:
    """[..., T, 64] logical rows -> the stored layout."""
    idx = _swz_index(rows.shape[-2]).expand(rows.shape)
    return torch.empty_like(rows).scatter_(-1, idx, rows)


def unswizzle(stored: torch.Tensor) -> torch.Tensor:
    idx = _swz_index(stored.shape[-2]).to(stored.device).expand(stored.shape)
    return stored.gather(-1, idx)


# ---- rotary embedding in the model dtype --------------------------------------------------------------------------------
def rope_tables(dtype, n_pos=MAX_POS + 1, theta=10000.0):
    """ParlerTTSRotaryEmbedding's fp32 cos / sin rows, in the model dtype (one spare row for the off-by-one bug model)."""
    inv = 1.0 / (theta ** (torch.arange(0, HD, 2, dtype=torch.int64).float() / HD))
    fr = torch.arange(n_pos, dtype=torch.int64).float()[:, None] * inv[None, :]
    emb = torch.cat((fr, fr), dim=-1)
    return emb.cos().to(dtype), emb.sin().to(dtype)


def rope(x: torch.Tensor, pos: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """apply_rotary_pos_emb in x's dtype: every product and the sum rounded to it.  x [..., 64], pos broadcast to x[..., 0]."""
    c, s = cos[pos], sin[pos]
    rot = torch.cat((-x[..., HD // 2:], x[..., : HD // 2]), dim=-1)
    return x * c + rot * s


# ---- cases --------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Case:
    dtype: torch.dtype
    B: int
    nh: int
    nkv: int
    q_len: int
    past: int
    cross: bool
    kv_len: int
    cap: int
    rope: bool
    qkv: torch.Tensor                 # self [B*q_len, (nh+2nkv)*64] | cross [B*q_len, nh*64]
    kc: torch.Tensor                  # [B, nkv, cap, 64] logical rows before the call
    vc: torch.Tensor
    mask: torch.Tensor | None         # int32 [B, mask_len]
    ch: int                           # keys per chunk of the sweep (bug models)
    needle: list                      # per row: the planted key index or -1
    plan: list                        # (pattern, row, [bug, ...])
    zero_rows: list                   # rows whose output must be exactly 0 (cross, fully masked, zero K/V)
    sweep: int = 0                    # prefill_sweep argument of the hook

    @property
    def rep(self):
        return self.nh // self.nkv

    def q_raw(self):
        return self.qkv[:, : self.nh * HD].view(self.B, self.q_len, self.nh, HD)

    def positions(self, shift=0):
        return torch.arange(self.past, self.past + self.q_len) + shift


def _distinct(sign: float, dtype):
    d = torch.arange(HD)
    return (sign * torch.where(d % 2 == 0, 3.0, -2.0)).to(dtype)


def _align(q_rot: torch.Tensor, score: float) -> torch.Tensor:
    """A key row whose score q.k/8 against q_rot (float) is `score`."""
    q = q_rot.double()
    return q * (score * 8.0 / float(q @ q))


def _query_heads(g, B, q_len, nh, share: bool, hi_freq: bool):
    """Raw query rows.  share: one vector per (row, head) for every position (prefill: a needle then stands out for all
    queries); the energy sits in the lowest rotary frequencies then, so that rotation between positions barely moves the
    scores.  hi_freq: energy in the highest frequencies (a one-position rotary shift then changes scores a lot)."""
    w = torch.full((HD,), 0.3, dtype=torch.float64)
    if share:
        w[[HD // 2 - 1, HD - 1, HD // 2 - 2, HD - 2]] = 3.0
    elif hi_freq:
        w[[0, 1, 2, 3, 32, 33, 34, 35]] = 3.0
    else:
        w[:] = 1.0
    n = 1 if share else q_len
    q = torch.randn(B, n, nh, HD, generator=g, dtype=torch.float64) * w
    return q.expand(B, q_len, nh, HD)


def make_case(kind: str, n: int, dtype, idx: int, sweep: int = 0, q_len: int = 1) -> Case:
    """kind: 'decode_self' (n cached keys + the step's own), 'decode_cross' (kv_len = n), 'prefill_self' (q_len = n, from
    position 0), 'prefill_cross' (kv_len = n encoder positions, q_len queries)."""
    g = torch.Generator().manual_seed(7919 * idx + n + (0 if dtype == torch.bfloat16 else 17))
    cross = kind.endswith("cross")
    decode = kind.startswith("decode")
    B = BATCHES[idx % 3]
    if cross:
        nh, nkv = [(4, 1), (4, 4), (8, 1), (2, 2)][idx % 4]
    else:
        nh, nkv = [(4, 4), (4, 2), (4, 1), (8, 2), (2, 2)][idx % 5]
    if sweep == 0 and not decode and dtype == torch.bfloat16:
        nkv = nh                               # the tensor-core prefill sweep is the bf16 MHA path
    if decode:
        q_len = 1
    elif not cross:
        q_len = n
    rope_on = idx % 3 != 2
    has_mask = idx % 4 != 3
    if decode:
        past = n if not cross else MAX_POS - 1 - (idx % 7)
        ch = 32 if dtype == torch.bfloat16 else 16
    else:
        past = 0 if (not cross or idx % 2 == 0) else MAX_POS - q_len
        ch = 32
    n_keys = n  # cached keys (self decode) / encoder keys (cross) / prompt+BOS keys (prefill self)
    cap = (past + q_len if not cross else n) + 3
    if B * nkv * cap > 6_000_000 or (not decode and max(n, q_len) >= 257):
        B = min(B, 5)   # (host memory and the cost of the float64 reference)
    cos, sin = rope_tables(dtype)

    share = not decode
    q = _query_heads(g, B, q_len, nh, share=share, hi_freq=decode)
    if cross:
        qkv = q.reshape(B * q_len, nh * HD).to(dtype)
    else:
        knew = torch.randn(B, q_len, nkv, HD, generator=g, dtype=torch.float64) * 0.5
        vnew = torch.randn(B, q_len, nkv, HD, generator=g, dtype=torch.float64)
        qkv = torch.cat((q.reshape(B * q_len, nh * HD), knew.reshape(B * q_len, nkv * HD), vnew.reshape(B * q_len, nkv * HD)),
                        dim=1).to(dtype)
    kc = torch.zeros(B, nkv, cap, HD, dtype=dtype)
    vc = torch.zeros(B, nkv, cap, HD, dtype=dtype)
    if decode or cross:
        kc[:, :, :n_keys] = (torch.randn(B, nkv, n_keys, HD, generator=g) * 0.5).to(dtype)
        vc[:, :, :n_keys] = torch.randn(B, nkv, n_keys, HD, generator=g).to(dtype)

    # masks: a left-padded prompt (self: mask_len < n keys) or description (cross: mask_len = S) per row
    mask = None
    mask_len = 0
    pads = [0] * B
    if has_mask:
        mask_len = n_keys if cross else (max(1, n_keys // 2) if decode else n_keys - 1)
        if mask_len > 0:
            mask = torch.ones(B, mask_len, dtype=torch.int32)
            for b in range(B):
                pads[b] = int(torch.randint(0, max(1, mask_len // 2) + 1, (1,), generator=g))
                mask[b, : pads[b]] = 0

    if decode and not cross:
        patterns = ["needle0", "needle_first", "needle_last", "needle_warp1", "needle_tail", "needle_own", "masked_needle",
                    "rising", "falling", "spread", "rope_decoy"]
    elif decode:
        patterns = ["needle0", "needle_first", "needle_last", "needle_warp1", "needle_tail", "masked_needle", "rising",
                    "falling", "spread", "rope_decoy", "fully_masked"]
    elif cross:
        patterns = ["needle0", "needle_first", "needle_last", "needle_tail", "masked_needle", "rising", "falling", "spread",
                    "fully_masked"]
    else:
        patterns = ["needle0", "needle_first", "needle_last", "needle_tail", "masked_needle", "rising", "falling", "spread"]

    q_rot = rope(q.to(dtype), past + torch.arange(q_len)[None, :, None], cos, sin) if rope_on else q.to(dtype)
    needle, plan, zero_rows = [-1] * B, [], []
    n_chunks = (n_keys + ch - 1) // ch
    for b in range(B):
        pat = patterns[(b + idx) % len(patterns)]
        if pat in ("rising", "falling") and n_chunks < 3:
            pat = "needle_tail"
        if pat == "masked_needle" and (mask is None or mask_len < 2):
            pat = "needle0"
        if pat == "rope_decoy" and (not rope_on or n_keys < 2):
            pat = "needle_first"
        if pat == "fully_masked" and mask is None:
            pat = "needle_last"
        if pat == "needle_own" and cross:
            pat = "needle_tail"
        t_of = {"needle0": 0, "needle_first": ch * (n_chunks // 2), "needle_last": ch * max(1, n_chunks // 2) - 1,
                "needle_warp1": ch + ch // 2, "needle_tail": n_keys - 1, "spread": None}
        bugs: list = []
        vdist = _distinct(1.0, dtype)
        for kvh in range(nkv):
            h0 = kvh * (nh // nkv)                     # planted against the group's first query head
            qr = q_rot[b, -1, h0].double()             # ... and its last position (decode: the only one)
            if pat in t_of and pat != "spread":
                t = min(t_of[pat], n_keys - 1)
                if not (decode or cross):             # prefill self: the key appended at position t, rotated by the kernel
                    knew_row = _align(q[b, 0, h0], GAP)
                    qkv[b * q_len + t, (nh + kvh) * HD:(nh + kvh + 1) * HD] = knew_row.to(dtype)
                    qkv[b * q_len + t, (nh + nkv + kvh) * HD:(nh + nkv + kvh + 1) * HD] = vdist
                else:
                    kc[b, kvh, t] = _align(qr, GAP).to(dtype)
                    vc[b, kvh, t] = vdist
                needle[b] = t
                if mask is not None and t < mask_len:
                    mask[b, t] = 1
            elif pat == "needle_own":
                qkv[b, (nh + kvh) * HD:(nh + kvh + 1) * HD] = _align(q[b, 0, h0], GAP).to(dtype)
                qkv[b, (nh + nkv + kvh) * HD:(nh + nkv + kvh + 1) * HD] = vdist
                needle[b] = past
            elif pat == "masked_needle":
                pads[b] = max(pads[b], 1, mask_len // 2)
                mask[b, : pads[b]] = 0
                t = pads[b] - 1
                if decode or cross:
                    kc[b, kvh, t] = _align(qr, GAP).to(dtype)
                    vc[b, kvh, t] = vdist
                else:
                    qkv[b * q_len + t, (nh + kvh) * HD:(nh + kvh + 1) * HD] = _align(q[b, 0, h0], GAP).to(dtype)
                    qkv[b * q_len + t, (nh + nkv + kvh) * HD:(nh + nkv + kvh + 1) * HD] = vdist
            elif pat in ("rising", "falling", "spread"):
                if pat == "spread":
                    a = torch.rand(n_keys, generator=g, dtype=torch.float64) * 110.0 - 110.0
                    t = int(torch.randint(0, n_keys, (1,), generator=g))
                    a[t] = 10.0
                    needle[b] = t
                    if mask is not None and t < mask_len:
                        mask[b, t] = 1
                else:
                    a = torch.linspace(-100.0, 10.0, n_keys, dtype=torch.float64)
                    if pat == "falling":
                        a = a.flip(0)
                        if mask is not None:   # (no padding: the top keys are the first ones)
                            mask[b] = 1
                base = q[b, 0, h0] if not (decode or cross) else qr
                rows = a[:, None] * _align(base, 1.0)[None, :]
                rows = rows + 0.02 * torch.randn(n_keys, HD, generator=g, dtype=torch.float64)
                if decode or cross:
                    kc[b, kvh, :n_keys] = rows.to(dtype)
                else:
                    qkv[b * q_len:(b + 1) * q_len, (nh + kvh) * HD:(nh + kvh + 1) * HD] = rows.to(dtype)
            elif pat == "rope_decoy":
                t1, t2 = n_keys - 1, n_keys // 2 if n_keys // 2 != n_keys - 1 else 0
                kc[b, kvh, t1] = _align(qr, GAP).to(dtype)
                vc[b, kvh, t1] = vdist
                q_shift = rope(q[b, 0, h0].to(dtype), torch.tensor(past + 1), cos, sin).double()
                kc[b, kvh, t2] = _align(q_shift, GAP).to(dtype)
                vc[b, kvh, t2] = _distinct(-1.0, dtype)
                if mask is not None:
                    mask[b, [t for t in (t1, t2) if t < mask_len]] = 1
            elif pat == "fully_masked":
                mask[b, :] = 0
                kc[b, :, :n_keys] = 0
                vc[b, :, :n_keys] = 0
        if cross and mask is not None and pat != "masked_needle":   # quirk Q8: masked encoder states are zero, so are their K/V
            off = (mask[b] == 0).nonzero().flatten()
            kc[b, :, off] = 0
            vc[b, :, off] = 0
        if pat.startswith("needle") or pat == "spread":
            bugs = ["drop_needle"]
            if pat == "needle_own":
                bugs = ["omit_own"]
            if pat == "needle_tail" and decode and n_keys % ch != 0:
                bugs.append("drop_tail")
        elif pat == "masked_needle":
            bugs = ["ignore_mask"]
        elif pat == "rising":
            bugs = ["no_rescale"]
        elif pat == "falling":
            bugs = ["drop_first_chunk"]
        elif pat == "rope_decoy":
            bugs = ["rope_shift"]
        elif pat == "fully_masked":
            zero_rows.append(b)
        plan.append((pat, b, bugs))
    return Case(dtype=dtype, B=B, nh=nh, nkv=nkv, q_len=q_len, past=past, cross=cross, kv_len=n if cross else 0, cap=cap,
                rope=rope_on, qkv=qkv, kc=kc, vc=vc, mask=mask, ch=ch, needle=needle, plan=plan, zero_rows=zero_rows,
                sweep=sweep)


# ---- the float64 reference ----------------------------------------------------------------------------------------------
def appended_rows(c: Case, shift: int = 0):
    """The K (rotated, model dtype) and V rows a self-attention call appends at positions past .. past + q_len - 1."""
    nh, nkv = c.nh, c.nkv
    k = c.qkv[:, nh * HD:(nh + nkv) * HD].view(c.B, c.q_len, nkv, HD)
    v = c.qkv[:, (nh + nkv) * HD:].view(c.B, c.q_len, nkv, HD)
    if c.rope:
        cos, sin = rope_tables(c.dtype)
        k = rope(k, c.positions(shift)[None, :, None], cos, sin)
    return k.permute(0, 2, 1, 3), v.permute(0, 2, 1, 3)   # [B, nkv, q_len, 64]


def k_cache_slack(c: Case) -> torch.Tensor:
    """Allowed |kernel - torch| per element of the K cache [B, nkv, cap, 64]: 0 (bit for bit) except for the rows an fp32
    rotary call appends, where the kernel may contract x*cos + rotate_half(x)*sin into one fma (one rounding fewer than
    torch): 2 ulp of the larger term."""
    slack = torch.zeros(c.kc.shape, dtype=torch.float64)
    if c.cross or not c.rope or c.dtype != torch.float32:
        return slack
    cos, sin = rope_tables(torch.float32)
    x = c.qkv[:, c.nh * HD:(c.nh + c.nkv) * HD].view(c.B, c.q_len, c.nkv, HD).double()
    pos = c.positions()[None, :, None]
    rot = torch.cat((-x[..., HD // 2:], x[..., : HD // 2]), dim=-1)
    terms = (x * cos[pos].double()).abs() + (rot * sin[pos].double()).abs()
    slack[:, :, c.past:c.past + c.q_len] = 2.0 ** -22 * terms.permute(0, 2, 1, 3)
    return slack


def assert_k_cache(got: torch.Tensor, want: torch.Tensor, slack: torch.Tensor):
    if want.dtype == torch.bfloat16:
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), "K cache rows differ from the bf16 rotary"
    else:
        err = (got.double() - want.double()).abs()
        assert bool((err <= slack).all()), f"K cache rows differ from the fp32 rotary by up to {float((err - slack).max()):.3g} " \
            "beyond one fma contraction"


def reference(c: Case, bug: str | None = None):
    """float64 softmax(q K^T / 8) V of every (row, position, head) -> (out, sum_i p_i |v_i|, attended) with out / mass
    [B*q_len, nh*64] and attended [B*q_len] (False: every key of the query is masked)."""
    shift = 1 if bug == "rope_shift" else 0
    q = c.q_raw()
    if c.rope:
        cos, sin = rope_tables(c.dtype)
        q = rope(q, c.positions(shift)[None, :, None], cos, sin)
    q = q.double()
    K, V = c.kc.double().clone(), c.vc.double().clone()
    if not c.cross:
        k_new, v_new = appended_rows(c, shift)
        K[:, :, c.past:c.past + c.q_len] = k_new.double()
        V[:, :, c.past:c.past + c.q_len] = v_new.double()
    T = c.kv_len if c.cross else c.past + c.q_len
    K, V = K[:, :, :T], V[:, :, :T]
    out = torch.zeros(c.B, c.q_len, c.nh, HD, dtype=torch.float64)
    mass = torch.zeros_like(out)
    attended = torch.ones(c.B, c.q_len, dtype=torch.bool)
    t = torch.arange(T)
    n_cached = c.kv_len if c.cross else c.past   # keys that come from the cache (decode: all but the own key)
    for b in range(c.B):
        keep = torch.ones(c.q_len, T, dtype=torch.bool)
        if not c.cross:
            keep &= t[None, :] <= c.positions()[:, None]
        if c.mask is not None and bug != "ignore_mask":
            ml = c.mask.shape[1]
            keep[:, :ml] &= (c.mask[b] != 0)[None, :]
        if bug == "drop_needle" and c.needle[b] >= 0:
            keep[:, c.needle[b]] = False
        if bug == "omit_own":
            keep &= t[None, :] != c.positions()[:, None]
        if bug == "drop_tail" and n_cached % c.ch:
            keep[:, (n_cached // c.ch) * c.ch:n_cached] = False
        if bug == "drop_first_chunk":
            keep[:, : c.ch] = False
        attended[b] = keep.any(1)
        for h in range(c.nh):
            kvh = h // c.rep
            s = (q[b, :, h] @ K[b, kvh].T) / 8.0
            s = s.masked_fill(~keep, -math.inf)
            if bug == "no_rescale":   # every chunk's terms stay scaled by the running maximum they were added under
                nch = (T + c.ch - 1) // c.ch
                sp = torch.full((c.q_len, nch * c.ch), -math.inf, dtype=torch.float64)
                sp[:, :T] = s
                m = sp.view(c.q_len, nch, c.ch).max(-1).values.cummax(1).values.repeat_interleave(c.ch, 1)[:, :T]
            else:
                m = s.max(1, keepdim=True).values.expand_as(s)
            m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
            w = torch.exp(s - m)
            l = w.sum(1, keepdim=True)
            p = torch.where(l > 0, w / torch.where(l > 0, l, torch.ones_like(l)), torch.zeros_like(w))
            out[b, :, h] = p @ V[b, kvh]
            mass[b, :, h] = p @ V[b, kvh].abs()
    return out.view(c.B * c.q_len, c.nh * HD), mass.view(c.B * c.q_len, c.nh * HD), attended.view(-1)


def bar(c: Case, ref: torch.Tensor, mass: torch.Tensor) -> torch.Tensor:
    if c.dtype == torch.bfloat16:
        return 2.0 ** -8 * (ref.abs() + mass) + 1e-6
    return 1e-5 * mass


def _rows_of(c: Case, b: int) -> slice:
    return slice(b * c.q_len, (b + 1) * c.q_len)


# ---- parametrisation ----------------------------------------------------------------------------------------------------
DTYPES = {"bf16": torch.bfloat16, "f32": torch.float32}
DECODE_IDS = [(kind, n, dt) for kind in ("decode_self", "decode_cross") for n in DECODE_N for dt in DTYPES]
PREFILL_IDS = ([("prefill_self", n, "bf16", 0) for n in PREFILL_Q] + [("prefill_self", n, dt, 1) for n in PREFILL_Q for dt in DTYPES]
               + [("prefill_cross", n, "bf16", 0) for n in CROSS_S] + [("prefill_cross", n, dt, 1) for n in CROSS_S for dt in DTYPES])


def _decode_case(kind, n, dt):
    return make_case(kind, n, DTYPES[dt], DECODE_N.index(n) + (0 if kind == "decode_self" else 1))


def _prefill_case(kind, n, dt, sweep):
    idx = (PREFILL_Q if kind == "prefill_self" else CROSS_S).index(n) + sweep
    return make_case(kind, n, DTYPES[dt], idx, sweep=sweep, q_len=(9, 33)[idx % 2])


ALL_CASES = [("decode",) + p for p in DECODE_IDS] + [("prefill",) + p for p in PREFILL_IDS]


def _build(p):
    return _decode_case(*p[1:]) if p[0] == "decode" else _prefill_case(*p[1:])


def _case_id(p):
    if p[0] == "decode":
        return f"{p[1]}-n{p[2]}-{p[3]}"
    return f"{p[1]}-n{p[2]}-{p[3]}-{'tc' if p[4] == 0 else 'item'}"


# ---- host tests: the reference, the layout helpers and the sensitivity of every planted case ---------------------------
def test_kv_swz_is_a_per_row_permutation_of_the_8_element_chunks():
    rows = torch.arange(37 * HD, dtype=torch.float32).view(37, HD)
    st = swizzle(rows)
    assert torch.equal(unswizzle(st), rows)
    for t in (0, 1, 7, 8, 36):
        assert sorted(st[t].tolist()) == rows[t].tolist()
        for d in range(HD):
            assert st[t, kv_swz(t, d)] == rows[t, d]
    assert torch.equal(st[8], rows[8]) and not torch.equal(st[9], rows[9])


def test_bf16_rope_rounds_every_product_and_the_sum():
    cos, sin = rope_tables(torch.bfloat16)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(50, HD, generator=g).to(torch.bfloat16)
    pos = torch.randint(0, MAX_POS, (50,), generator=g)
    got = rope(x, pos, cos, sin)
    xf, c, s = x.float(), cos[pos].float(), sin[pos].float()
    rot = torch.cat((-xf[:, 32:], xf[:, :32]), -1)
    r = lambda a: a.to(torch.bfloat16).float()
    assert torch.equal(got.float(), r(r(xf * c) + r(rot * s)))


@pytest.mark.parametrize("gqa", [False, True])
@pytest.mark.parametrize("cross", [False, True])
def test_reference_equals_torch_sdpa(cross, gqa):
    """The float64 reference against F.scaled_dot_product_attention (float64, boolean masks, repeated K/V heads)."""
    nh, nkv = (4, 2) if gqa else (2, 2)
    B, q_len, past, S = 3, 5, 6, 9
    g = torch.Generator().manual_seed(11)
    cos, sin = rope_tables(torch.float32)
    T = S if cross else past + q_len
    W = nh * HD if cross else (nh + 2 * nkv) * HD
    qkv = torch.randn(B * q_len, W, generator=g)
    kc = torch.zeros(B, nkv, T + 2, HD)
    vc = torch.zeros(B, nkv, T + 2, HD)
    n0 = S if cross else past
    kc[:, :, :n0] = torch.randn(B, nkv, n0, HD, generator=g)
    vc[:, :, :n0] = torch.randn(B, nkv, n0, HD, generator=g)
    mask = torch.ones(B, 4, dtype=torch.int32)
    mask[1, :2] = 0
    mask[2, 3] = 0
    c = Case(dtype=torch.float32, B=B, nh=nh, nkv=nkv, q_len=q_len, past=past, cross=cross, kv_len=S if cross else 0,
             cap=T + 2, rope=True, qkv=qkv, kc=kc, vc=vc, mask=mask, ch=16, needle=[-1] * B, plan=[], zero_rows=[])
    out, _, att = reference(c)
    assert att.all()
    q = rope(c.q_raw(), c.positions()[None, :, None], cos, sin).double().permute(0, 2, 1, 3)   # [B, nh, q, 64]
    K, V = kc.double().clone(), vc.double().clone()
    if not cross:
        k_new, v_new = appended_rows(c)
        K[:, :, past:past + q_len], V[:, :, past:past + q_len] = k_new.double(), v_new.double()
    K, V = K[:, :, :T].repeat_interleave(nh // nkv, 1), V[:, :, :T].repeat_interleave(nh // nkv, 1)
    allow = torch.ones(B, 1, q_len, T, dtype=torch.bool)
    allow[:, 0, :, :4] &= (mask != 0)[:, None, :]
    if not cross:
        allow &= torch.arange(T)[None, None, None, :] <= (past + torch.arange(q_len))[None, None, :, None]
    want = torch.nn.functional.scaled_dot_product_attention(q, K, V, attn_mask=allow, scale=0.125)
    want = want.permute(0, 2, 1, 3).reshape(B * q_len, nh * HD)
    assert torch.allclose(out, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("p", ALL_CASES, ids=[_case_id(p) for p in ALL_CASES])
def test_planted_case_sees_the_modelled_kernel_bugs(p):
    """Host side of every GPU case: each planted row moves by > 4x its bar under each bug it is meant to catch."""
    c = _build(p)
    ref, mass, att = reference(c)
    lim = bar(c, ref, mass)
    checked = 0
    for pat, b, bugs in c.plan:
        rows = _rows_of(c, b)
        ok = att[rows]
        for bug in bugs:
            alt, _, _ = reference(c, bug)   # (a query left with no key at all: 0, what the decode and tensor-core sweeps write)
            ratio = ((alt[rows] - ref[rows]).abs() / lim[rows])[ok]
            assert ratio.numel() > 0 and float(ratio.max()) > 4.0, f"row {b} ({pat}): bug {bug} moves the output by only " \
                f"{float(ratio.max()) if ratio.numel() else 0:.2f}x the bar"
            checked += 1
    assert checked > 0 or all(pat == "fully_masked" for pat, _, _ in c.plan)


# ---- the kernels ----------------------------------------------------------------------------------------------------------
def run_kernel(c: Case):
    from parler_tts_b200 import _lib
    dev = "cuda"
    dt = _lib.dtype_code(c.dtype)
    qkv = c.qkv.to(dev).contiguous()
    kc = swizzle(c.kc).to(dev).contiguous()
    vc = swizzle(c.vc).to(dev).contiguous()
    cos, sin = rope_tables(c.dtype)
    cos, sin = cos.to(dev).contiguous(), sin.to(dev).contiguous()
    mask = None if c.mask is None else c.mask.to(dev).contiguous()
    out = torch.full((c.B * c.q_len, c.nh * HD), float("nan"), dtype=c.dtype, device=dev)
    _lib.check(_lib.lib().ptts_op_attention(dt, c.B, c.nh, c.nkv, c.q_len, c.past, int(c.cross), c.kv_len, c.cap, int(c.rope),
                                            _lib.ptr(cos), _lib.ptr(sin), _lib.ptr(qkv), _lib.ptr(kc), _lib.ptr(vc), _lib.ptr(mask),
                                            0 if mask is None else mask.shape[1], c.sweep, _lib.ptr(out), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return out.cpu(), unswizzle(kc.cpu()), unswizzle(vc.cpu())


def check_against_reference(c: Case, record_property=None):
    got, kc, vc = run_kernel(c)
    assert torch.isfinite(got.float()).all(), "non-finite attention output"
    # cache contents: the appended rows are torch's model-dtype rotary of the new K and the new V; nothing else changed
    want_k, want_v = c.kc.clone(), c.vc.clone()
    if not c.cross:
        k_new, v_new = appended_rows(c)
        want_k[:, :, c.past:c.past + c.q_len] = k_new
        want_v[:, :, c.past:c.past + c.q_len] = v_new
    assert torch.equal(vc.view(torch.int16) if c.dtype == torch.bfloat16 else vc.view(torch.int32),
                       want_v.view(torch.int16) if c.dtype == torch.bfloat16 else want_v.view(torch.int32)), "V cache rows differ"
    assert_k_cache(kc, want_k, k_cache_slack(c))
    ref, mass, att = reference(c)
    lim = bar(c, ref, mass)
    err = (got.double() - ref).abs()
    ratio = (err / lim)[att]
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if record_property is not None:
        record_property("worst_error_to_bar", worst)
    bad = ((err / lim > 1.0) & att[:, None]).nonzero()[:5].tolist()
    assert worst <= 1.0, f"error {worst:.3g}x the bar; first offending (output row, column): {bad}; planted rows {c.plan}"
    for b in c.zero_rows:   # fully masked description row with zeroed K/V (quirk Q8): exactly 0
        assert torch.equal(got[_rows_of(c, b)].float(), torch.zeros_like(got[_rows_of(c, b)].float()))
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n,dt", DECODE_IDS, ids=[f"{k}-n{n}-{d}" for k, n, d in DECODE_IDS])
def test_decode_sweep_against_fp64(kind, n, dt, record_property):
    check_against_reference(_decode_case(kind, n, dt), record_property)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n,dt,sweep", PREFILL_IDS,
                         ids=[f"{k}-n{n}-{d}-{'tc' if s == 0 else 'item'}" for k, n, d, s in PREFILL_IDS])
def test_prefill_sweep_against_fp64(kind, n, dt, sweep, record_property):
    check_against_reference(_prefill_case(kind, n, dt, sweep), record_property)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,sweep", [("bf16", 0), ("bf16", 1), ("f32", 1)], ids=["bf16-tc", "bf16-item", "f32-item"])
def test_prefill_then_decode_appends_up_to_position_4095(dt, sweep):
    """A 33-position prefill, then single-position decode calls at positions 33 .. 40 and 4088 .. 4095 on the same caches:
    every row the kernels wrote reads back as the model-dtype rotary of its K and its V, bit for bit (bf16), and every
    output stays within the bar."""
    from parler_tts_b200 import _lib
    dtype = DTYPES[dt]
    cos, sin = rope_tables(dtype)
    g = torch.Generator().manual_seed(5)
    B, nh, nkv, P1, cap = 3, 4, 4 if sweep == 0 else 2, 33, MAX_POS
    kc = torch.zeros(B, nkv, cap, HD, dtype=dtype, device="cuda")
    vc = torch.zeros_like(kc)
    want_k = torch.zeros(B, nkv, cap, HD, dtype=dtype)
    want_v = torch.zeros_like(want_k)
    slack = torch.zeros(want_k.shape, dtype=torch.float64)
    steps =[(0, P1)] + [(p, 1) for p in list(range(P1, P1 + 8)) + list(range(MAX_POS - 8, MAX_POS))]
    worst = 0.0
    for past, q_len in steps:
        qkv = (torch.randn(B * q_len, (nh + 2 * nkv) * HD, generator=g)).to(dtype)
        c = Case(dtype=dtype, B=B, nh=nh, nkv=nkv, q_len=q_len, past=past, cross=False, kv_len=0, cap=cap, rope=True,
                 qkv=qkv, kc=want_k.clone(), vc=want_v.clone(), mask=None, ch=32, needle=[-1] * B, plan=[], zero_rows=[],
                 sweep=sweep)
        out = torch.empty(B * q_len, nh * HD, dtype=dtype, device="cuda")
        qd, cd, sd = qkv.cuda(), cos.cuda(), sin.cuda()
        _lib.check(_lib.lib().ptts_op_attention(_lib.dtype_code(dtype), B, nh, nkv, q_len, past, 0, 0, cap, 1, _lib.ptr(cd),
                                                _lib.ptr(sd), _lib.ptr(qd), _lib.ptr(kc), _lib.ptr(vc), None, 0, sweep,
                                                _lib.ptr(out), _lib.stream_ptr()))
        torch.cuda.synchronize()
        ref, mass, _ = reference(c)
        worst = max(worst, float(((out.cpu().double() - ref).abs() / bar(c, ref, mass)).max()))
        k_new, v_new = appended_rows(c)
        want_k[:, :, past:past + q_len] = k_new
        want_v[:, :, past:past + q_len] = v_new
        slack += k_cache_slack(c)
    got_k, got_v = unswizzle(kc.cpu()), unswizzle(vc.cpu())
    assert_k_cache(got_k, want_k, slack)
    assert torch.equal(got_v, want_v)
    assert worst <= 1.0, f"error {worst:.3g}x the bar"
