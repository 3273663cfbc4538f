"""The device sampler (sample_core.cuh) against a float64 reference of one sampler call and a host replica of its Philox stream.

Host part: the replica against the Random123 Philox4x32-10 known-answer vectors, the reference against oracle/sampling.py
(pinned to transformers) and tests/sampling_ext_oracle.py, and every modelled kernel bug moving the expected outcome of at least
one designed case.  GPU part: crafted logit rows written into a session's logits, one sampler call each, at vocabulary sizes that
run every ITEMS instantiation (1, 5, 9) with full slots and slots that end just past a slot edge (vocab_size is a multiple of 8,
so "one id over" is 8 ids over), through ptts_sample (plain and EXT kernels) and ptts_op_sample_phase (the step kernels'
three-row passes); then the logits of a bf16 Mini-shaped model, full of ties.

The reference, per row, in the kernel's order:
  1. MinNewTokens, ParlerTTSLogitsProcessor, the suppress_special mask and the n-gram bans: -inf;
  2. temperature (float32 v / float32 T, as the kernel divides), top-k (every id tied with the k-th value stays), top-p, then
     MinP, Typical, Epsilon and Eta, in float64 on p = exp(v - max) / S;
  3. the draw: the first id in index order whose cumulative mass exceeds u * S among ids with p > 0 (the last such id if none
     does), u = Philox4x32-10 of counter (row_base + row, column, 0x5054, 0x5453) and key (seed low word, seed high word),
     (c0 >> 8) * 2^-24; greedy: argmax, the smallest index on ties.
Top-p removes id i iff the mass of the ids scoring <= v_i is <= (1 - top_p) * S and v_i is not the max: a tie group goes or
stays as a whole (transformers' sorted-position rule can split it; the device keeps the whole group).
"""
from __future__ import annotations

import copy
import math

import numpy as np
import pytest
import torch

from oracle.config import mini_cfg, tiny_cfg
from oracle.sampling import ParlerLogitsProcessorOracle
from oracle import sampling as osamp
from tests import sampling_ext_oracle as so

DEV = "cuda"
SLOT = 256                                   # ids per slot: element i of a row lives on thread i % 256, slot i / 256
VOCABS = (96, 256, 264, 1088, 1280, 1288, 2304)  # ITEMS 1, 1, 2->5, 5, 5, 6->9, 9
B, K = 3, 4                                  # 12 rows per call (tiny_cfg has 4 codebooks)
EOS, PAD, BOS = 64, 64, 65                   # tiny_cfg's special ids
NEG = np.float32(-np.inf)
TOL_BAND = 1e-5                              # a draw whose u * S lies this close (relative to S) to a boundary may go either way
TOL_DESIGN = 1e-3                            # designed rows keep every threshold quantity this far (relative) from its threshold
TOL_REAL = 1e-6                              # realistic rows: a kept/removed decision this close to its threshold may flip
EXT_OFF = dict(no_repeat_ngram_size=0, min_p=0.0, typical_p=1.0, epsilon_cutoff=0.0, eta_cutoff=0.0)

# ---- Philox4x32-10 ----------------------------------------------------------------------------------------------------------
_M32 = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def philox4x32_10(ctr, key):
    """Random123's Philox4x32-10 on uint32 words (numpy, broadcast): ctr = 4 words, key = 2 words; returns 4 uint64 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & _M32 for x in ctr]
    k0, k1 = (np.asarray(k, dtype=np.uint64) & _M32 for k in key)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]   # < 2^64: the full 64-bit product
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> _S32) ^ c[1] ^ k0, p1 & _M32, (p0 >> _S32) ^ c[3] ^ k1, p0 & _M32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
    return c


def philox_uniform(seed: int, row, col, bug: str | None = None) -> np.ndarray:
    """philox_uniform(seed, row, col) of sample_core.cuh, in float64 (the float32 value is exact: 24 bits)."""
    seed = int(seed) & (2 ** 64 - 1)
    lo, hi = seed & 0xFFFFFFFF, seed >> 32
    if bug == "seed_lo":
        hi = 0
    if bug == "philox_swap":
        row, col = col, row
    row = np.asarray(row, dtype=np.int64).astype(np.uint64)
    col = np.asarray(col, dtype=np.int64).astype(np.uint64)
    c0 = philox4x32_10([row, col, 0x5054, 0x5453], [lo, hi])[0]
    return (c0 >> np.uint64(8)).astype(np.float64) * 2.0 ** -24


# Seeds found with the replica (test_special_seeds_put_u_where_the_cases_need_it checks them): for row row_base + 0 = 12345 at
# column 1, u < 2^-20, u > 1 - 2^-20, u * 64 = 60 exactly (a dyadic row of 64 ids then has u * S on a boundary), and
# u = 1 - 2^-23 (the largest but one; the fallback row below).
ENDS_ROW_BASE = 12345
SEED_LOW = 14210210037782985358
SEED_HIGH = 9323948316590194099
SEED_HIT = 18403911077917398051
SEED_TOP = 7550113450791922799

FALLBACK_IDS = (32, 33, 49)   # warp 1 of slot 0, lanes 0, 1 and 17


def fallback_row(V: int):
    """p = 1 at id 32 and e^-17 (< 2^-24 each, > 2^-24 together) at ids 33 and 49: the kernel's CTA sum adds the two small masses
    first (s = 1 + 2^-23), its scan adds each to 1 on its own (total 1), so with u = 1 - 2^-23 no cumulative sum exceeds u * s
    and the draw falls back to the last id with p > 0."""
    row = np.full(V, NEG, np.float32)
    row[list(FALLBACK_IDS)] = [0.0, -17.0, -17.0]
    return row


# ---- the reference -----------------------------------------------------------------------------------------------------------
BUGS = ("carry", "ge", "draw_order", "topk_ties", "topp_lt", "topp_positional", "argmax_last", "philox_swap", "no_row_base",
        "seed_lo", "temp_after_topp", "masks_after_topk", "no_last_id", "no_last_slot")
MULTI_SLOT_BUGS = ("carry", "draw_order")   # a one-slot row cannot show these


def _softmax(v):
    x = v.astype(np.float64)
    fin = np.isfinite(x)
    m = x[fin].max() if fin.any() else -np.inf
    e = np.zeros(x.size)
    e[fin] = np.exp(x[fin] - m)
    return x, m, e


def _groups(x, e, fin):
    vals, inv = np.unique(x[fin], return_inverse=True)
    gm = np.bincount(inv, weights=e[fin], minlength=vals.size)
    return vals, inv, np.cumsum(gm), gm


def sample_row(v, mask, g: dict, u: float, bug=None, tol=TOL_REAL):
    """One row: v float32 [V] (the raw logits), mask bool [V] (ids the EOS / special / n-gram masks remove).  Returns the
    processed float32 scores, the token, whether u * S lies within TOL_BAND * S of an inner boundary of the draw, and the ids
    whose kept/removed decision lies within tol (relative) of its threshold."""
    V = v.size
    near = np.zeros(V, bool)
    v = v.astype(np.float32).copy()
    if bug != "masks_after_topk":
        v[mask] = NEG
    if not g["do_sample"]:
        if bug == "masks_after_topk":
            v[mask] = NEG
        mx = v.max()
        tok = int(np.nonzero(v == mx)[0][-1 if bug == "argmax_last" else 0])
        return v, tok, False, near
    T = np.float32(g["temperature"])
    temper = (lambda a: a / T) if T != np.float32(1.0) else (lambda a: a)
    if bug != "temp_after_topp":
        v = temper(v)
    if g["top_k"] > 0:
        kk = min(g["top_k"], V)
        if bug == "topk_ties":
            keep = np.zeros(V, bool)
            keep[np.argsort(-v.astype(np.float64), kind="stable")[:kk]] = True
        else:
            keep = v >= np.sort(v)[V - kk]
        v = np.where(keep, v, NEG)
    if bug == "masks_after_topk":
        v[mask] = NEG
    x, m, e = _softmax(v)
    if g["top_p"] < 1.0:
        S = e.sum()
        bound = float(np.float32(1.0) - np.float32(g["top_p"])) * S
        fin = np.isfinite(x)
        rm = np.zeros(V, bool)
        if bug == "topp_positional":   # transformers: by position in the ascending (stable) sort
            order = np.argsort(x, kind="stable")
            r = np.cumsum(e[order]) <= bound
            r[-1] = False
            rm[order] = r
        else:
            vals, inv, le, gm = _groups(x, e, fin)
            rg = ((le - gm) if bug == "topp_lt" else le) <= bound
            rg[vals == m] = False
            rm[fin] = rg[inv]
            near[fin] |= ((np.abs(le - bound) <= tol * S) & (vals != m))[inv]
        v = np.where(rm, NEG, v)
        e = np.where(rm, 0.0, e)
    if bug == "temp_after_topp":
        v = temper(v)
        x, m, e = _softmax(v)
    ext = g.get("ext") or {}

    def drop(rm):
        nonlocal v, e
        v = np.where(rm, NEG, v)
        e = np.where(rm, 0.0, e)

    def entropy():
        x = v.astype(np.float64)
        fin = np.isfinite(x)
        lse = m + math.log(e.sum())
        lp = np.where(fin, x - lse, 0.0)
        return -(lp * np.exp(lp))[fin].sum(), lse, x, fin

    if ext.get("min_p", 0.0) > 0.0:                      # p < min_p * p_max, p_max = 1 / S
        thr = float(np.float32(ext["min_p"]))
        near |= np.isfinite(v) & (np.abs(e - thr) <= tol * thr)
        drop(e < thr)
    if ext.get("typical_p", 1.0) < 1.0:                  # keep shifted <= the first value whose mass reaches typical_p
        H, lse, x, fin = entropy()
        sh = np.where(fin, np.abs(lse - x - H), np.inf)
        target = float(np.float32(ext["typical_p"])) * e.sum()
        vals, inv, le, _ = _groups(sh, e, fin)
        near[fin] |= (np.abs(le - target) <= tol * e.sum())[inv]
        reach = np.nonzero(le >= target)[0]
        if reach.size:
            t = vals[reach[0]]
            near |= fin & (sh != t) & (np.abs(sh - t) <= tol * max(1.0, abs(t)))
            drop(fin & (sh > t))
    if 0.0 < ext.get("epsilon_cutoff", 0.0):
        eps = float(np.float32(ext["epsilon_cutoff"]))
        p = e / e.sum()
        near |= np.isfinite(v) & (v < m) & (np.abs(p - eps) <= tol * eps)
        drop((p < eps) & (v < m))
    if 0.0 < ext.get("eta_cutoff", 0.0):
        H, _, _, _ = entropy()
        eta = float(np.float32(ext["eta_cutoff"]))
        thr = min(eta, math.sqrt(eta) * math.exp(-H))
        p = e / e.sum()
        near |= np.isfinite(v) & (v < m) & (np.abs(p - thr) <= tol * thr)
        drop((p < thr) & (v < m))
    # the draw
    S = e.sum()
    ids = np.arange(V)
    order = np.lexsort((ids // SLOT, ids % SLOT)) if bug == "draw_order" else ids
    eo = e[order]
    cum = np.cumsum(eo)
    if bug == "carry":   # each slot's scan starts again from 0
        first = np.searchsorted(order // SLOT, order // SLOT)   # index order: the first position of each element's slot
        cum = cum - np.concatenate([[0.0], cum])[first]
    target = u * S
    live = eo > 0
    hit = ((cum >= target) if bug == "ge" else (cum > target)) & live
    nz = np.nonzero(live)[0]
    if hit.any():
        k = int(np.argmax(hit))
    elif nz.size:
        k = int(nz[-1])
    else:
        return v, 0, False, near
    j = int(np.searchsorted(nz, k))
    band = (j > 0 and target - cum[nz[j - 1]] < TOL_BAND * S) or (j < nz.size - 1 and cum[k] - target < TOL_BAND * S)
    return v, int(order[k]), bool(band), near


def mask_matrix(hist, g: dict, parler, V: int, bug=None):
    """The ids MinNewTokens, the Parler rule, suppress_special and the n-gram bans remove from each row, and the Parler state
    after this call."""
    R, cur = hist.shape
    z = np.zeros((R, V), np.float32)
    if cur - 1 < g.get("min_new_tokens", 0):
        z[:, g["eos"]] = -np.inf
    parler = copy.deepcopy(parler)
    z = parler(hist, z)
    if g.get("suppress_special"):
        z[:, g["codebook_size"]:] = -np.inf
    z = so.no_repeat_ngram(hist, z, int((g.get("ext") or {}).get("no_repeat_ngram_size", 0)))
    if bug == "no_last_id":
        z[:, V - 1] = -np.inf
    if bug == "no_last_slot":
        z[:, (V - 1) // SLOT * SLOT:] = -np.inf
    return np.isneginf(z), parler


def reference_call(logits, hist, g: dict, parler, unfinished, cur: int, forced=None, bug=None, tol=TOL_REAL):
    """One sampler call on rows [R, V] at column cur with the history hist [R, cur]."""
    R, V = logits.shape
    mask, parler = mask_matrix(hist, g, parler, V, bug)
    rows = np.arange(R) + (0 if bug == "no_row_base" else g["row_base"])
    u = philox_uniform(g["seed"], rows, cur, bug)
    scores = np.empty((R, V), np.float32)
    tok, band, near = np.zeros(R, np.int64), np.zeros(R, bool), np.zeros((R, V), bool)
    for r in range(R):
        scores[r], tok[r], band[r], near[r] = sample_row(logits[r], mask[r], g, float(u[r]), bug, tol)
    out = tok.copy() if forced is None else np.asarray(forced, np.int64).copy()
    out[~unfinished] = g["pad"]
    return dict(scores=scores, drawn=tok, token=out, band=band, near=near, parler=parler, u=u)


def simulate(group, V: int, bug=None, tol=TOL_REAL):
    """Every call of a designed group, each on the history the calls before it wrote."""
    g = group["gen"]
    R = B * K
    hist = np.full((R, 1), BOS, np.int64)
    parler = ParlerLogitsProcessorOracle(EOS, K, B)
    unf = np.ones(R, bool)
    res = []
    for call in group["calls"]:
        r = reference_call(call["rows"], hist, g, parler, unf, hist.shape[1], call.get("forced"), bug, tol)
        parler = r["parler"]
        hist = np.concatenate([hist, r["token"][:, None]], 1)
        unf &= r["token"] != EOS
        res.append(r)
    return res


# ---- designed cases -----------------------------------------------------------------------------------------------------------
STRADDLE = [0.01, 0.015, 0.02, 0.035, 0.035, 0.035, 0.06, 0.09, 0.12, 0.17, 0.41]   # ties at 0.035 span [0.045, 0.15]
PEAK2 = [0.5, 0.2, 0.15, 0.1, 0.05]
MAXTIE = [0.3, 0.3, 0.2, 0.1, 0.1]
TAIL = [0.001, 0.0025, 0.0215, 0.05, 0.1, 0.125, 0.2, 0.5]
MINP_ROW = [0.4, 0.2, 0.1, 0.03, 0.02, 0.25]


def edge_ids(V: int):
    """Ids at slot, warp and lane edges: 0, 31, 32, 255, 256, 256 j +- 1, V - 1 (EOS excluded: it stays -inf outside the mask
    cases)."""
    e = {0, 1, 31, 32, 33, 63, 95, 127, 128, 224, 255, V - 2, V - 1}
    for j in range(1, (V + SLOT - 1) // SLOT):
        e |= {SLOT * j - 1, SLOT * j, SLOT * j + 1, SLOT * j + 31, SLOT * j + 32}
    return sorted(i for i in e if 0 <= i < V and i != EOS)


def pick_ids(rng, V: int, n: int):
    """n distinct ids, edge ids first (in random order), then random others."""
    edges = list(rng.permutation(edge_ids(V)))
    taken = set(edges) | {EOS}
    rest = [i for i in rng.permutation(V) if i not in taken]
    return np.array((edges + rest)[:n], np.int64)


def spread3(V: int):
    """Three ids in different slots (or lanes far apart on a one-slot vocabulary)."""
    mid = SLOT + 1 if V > SLOT + 1 else V // 2 + 1
    return [31, mid, V - 1]


def mass_row(V, ids, masses, fill=-np.inf, T=1.0, eos=None):
    row = np.full(V, fill, np.float32)
    row[np.asarray(ids)] = (np.log(np.asarray(masses, np.float64)) * T).astype(np.float32)
    row[EOS] = NEG if eos is None else eos
    return row


def masses_at(rng, V, masses, tie_ids=None):
    """Ids for a mass pattern: the tied masses of STRADDLE / MAXTIE go to ids in different slots."""
    ids = list(pick_ids(rng, V, len(masses) + 3))
    if tie_ids is not None:
        for t in tie_ids:
            if t in ids:
                ids.remove(t)
        vals = np.asarray(masses)
        out = np.empty(len(masses), np.int64)
        tied = [i for i in range(len(masses)) if (vals == vals[i]).sum() == 3]
        for i, t in zip(tied, tie_ids):
            out[i] = t
        rest = [i for i in range(len(masses)) if i not in tied]
        out[rest] = ids[:len(rest)]
        return out
    return np.array(ids[:len(masses)])


def dyadic_row(rng, V, n, fill, value=2.5):
    row = np.full(V, fill, np.float32)
    row[pick_ids(rng, V, n)] = value
    row[EOS] = NEG
    return row


def gen(**kw):
    g = dict(do_sample=True, temperature=1.0, top_k=0, top_p=1.0, min_new_tokens=0, suppress_special=False, codebook_size=1024,
             ext=None, eos=EOS, pad=PAD, seed=2 ** 64 - 1, row_base=0)
    g.update(kw)
    return g


def _designed(V: int, name: str, rng, g: dict, row_fns, n_calls=2, exact=False, forced=None):
    R = B * K
    calls = []
    for c in range(n_calls):
        rows = np.stack([row_fns[r % len(row_fns)](rng, r) for r in range(R)])
        calls.append(dict(rows=rows, forced=None if forced is None else forced[c], exact=exact))
    return dict(name=name, gen=g, calls=calls)


def design_groups(V: int, ext: bool = True):
    """The designed groups of one vocabulary size (each = one generation: begin, prefill, then its calls)."""
    rng = np.random.default_rng(V)
    R = B * K
    out = []
    fills = (-np.inf, np.float32(-1e4))
    tie3 = spread3(V)
    n_max = 64

    def dy(rng, r):
        return dyadic_row(rng, V, 2 ** (r % 7), fills[r % 2])

    def all_edges(rng, r):   # every edge id live, a power of two of them
        ids = edge_ids(V)
        ids = ids[:2 ** int(math.log2(len(ids)))]
        row = np.full(V, fills[r % 2], np.float32)
        row[ids] = -1.75
        return row

    out.append(_designed(V, "dyadic", rng, gen(), [dy, dy, dy, all_edges], n_calls=3, exact=True))
    out.append(_designed(V, "dyadic_t07_topk", rng, gen(temperature=0.7, top_k=V + 5), [dy], n_calls=2, exact=True))

    def hit(rng, r):   # 64 equal ids: u * 64 = 60 exactly for row 0
        return dyadic_row(rng, V, n_max, fills[0]) if r == 0 else dy(rng, r)

    out.append(_designed(V, "dyadic_boundary", rng, gen(seed=SEED_HIT, row_base=ENDS_ROW_BASE), [hit], n_calls=1, exact=True))

    # top-k: the k-th value shared by ids in different slots; EOS finite and tied with the smallest values in full rows
    def topk_row(rng, r):
        row = (np.float32(-30.0) + np.round(rng.uniform(0, 4, V) * 8) / 8).astype(np.float32)   # tail: ties, mass ~1e-10
        low = pick_ids(rng, V, 3)
        row[low] = -30.0
        row[EOS] = -30.0
        if r % 3 == 1:
            row[rng.choice(V, V // 5, replace=False)] = NEG     # masked ids
            row[EOS] = NEG
        head = [i for i in pick_ids(rng, V, 12) if i not in tie3]
        vals = [6.0, 5.5, 5.25, 5.0, 4.0, 3.5, 3.25]
        row[head[:len(vals)]] = vals
        row[tie3] = 4.5                                        # the 5th value, three times
        if r % 4 == 3:
            row[head[0]] = 5.5                                  # a tie at the max
        return row

    for k in (1, 5, V - 1, V, V + 5):
        out.append(_designed(V, f"topk{k}", rng, gen(top_k=k), [topk_row], n_calls=2))
    # top-p
    def mrow(masses, T=1.0, tie=None):
        def f(rng, r):
            return mass_row(V, masses_at(rng, V, masses, tie), masses, fills[r % 2], T)
        return f

    def flat(rng, r):
        row = np.full(V, 1.25, np.float32)
        row[EOS] = NEG
        return row

    straddle = lambda T=1.0: mrow(STRADDLE, T, tie3)
    out.append(_designed(V, "topp0.9", rng, gen(top_p=0.9), [straddle(), mrow(MAXTIE), mrow(PEAK2), mrow(TAIL), flat]))
    out.append(_designed(V, "topp0.02", rng, gen(top_p=0.02), [mrow(PEAK2), mrow(MAXTIE), straddle(), flat]))
    out.append(_designed(V, "topp0.995", rng, gen(top_p=0.995), [mrow(TAIL), straddle(), mrow(PEAK2)]))
    for T in (0.05, 3.0):
        out.append(_designed(V, f"t{T}_topp0.9", rng, gen(temperature=T, top_p=0.9), [straddle(T), mrow(TAIL, T), mrow(MAXTIE, T)]))
        out.append(_designed(V, f"t{T}_topk6", rng, gen(temperature=T, top_k=6), [topk_row]))

    # peaked and extreme rows
    def peak(rng, r):
        row = rng.standard_normal(V).astype(np.float32)
        row[EOS] = NEG
        row[pick_ids(rng, V, 1)] = row.max() + 30.0
        return row

    def extreme(rng, r):
        row = (np.float32(-1e4) + np.round(rng.standard_normal(V) * 64) / 64).astype(np.float32)
        ids = masses_at(rng, V, TAIL)
        row[ids] = np.float32(1e4) + np.round(np.log(TAIL) * 64) / 64
        row[EOS] = NEG
        return row

    out.append(_designed(V, "peaked_extreme", rng, gen(), [peak, extreme]))
    # masks: EOS (or the special ids) hold the max while a rule masks them, with top-k after the masks
    def eos_max(k_rows):
        def f(rng, r):
            row = rng.standard_normal(V).astype(np.float32)
            head = pick_ids(rng, V, 5)
            row[head] = [8.0, 7.5, 7.25, 7.0, 6.5]
            row[EOS] = 9.0 if (r % K) in k_rows else NEG
            return row
        return f

    out.append(_designed(V, "min_new_tokens", rng, gen(top_k=3, min_new_tokens=100), [eos_max(range(K))]))
    out.append(_designed(V, "parler_rule", rng, gen(top_k=3), [eos_max(range(1, K))]))
    cb = 2 * V // 3

    def special(rng, r):
        row = rng.standard_normal(V).astype(np.float32)
        row[[cb, V - 1]] = [9.0, 8.5]
        row[[i for i in pick_ids(rng, V, 20) if i < cb][:4]] = [8.0, 7.5, 7.25, 7.0]
        row[EOS] = NEG
        return row

    out.append(_designed(V, "suppress_special", rng, gen(top_k=3, suppress_special=True, codebook_size=cb), [special]))

    # greedy
    def g_ties(rng, r):
        row = rng.standard_normal(V).astype(np.float32)
        row[EOS] = NEG
        kind = r % 5
        if kind == 0:
            row[tie3[::-1]] = 5.0                               # the max in three slots: the smallest index
        elif kind == 1:
            row[V - 1] = 5.0                                    # the max at V - 1
        elif kind == 2:
            row[:] = 0.5                                        # all equal: id 0
            row[EOS] = NEG
        elif kind == 3:
            row[[0, V - 1]] = 5.0
        else:
            row[EOS] = 9.0                                      # EOS masked by MinNewTokens
            row[V - 2] = 5.0
        return row

    out.append(_designed(V, "greedy", rng, gen(do_sample=False, min_new_tokens=100), [g_ties], n_calls=2))
    out.append(_designed(V, "greedy_parler", rng, gen(do_sample=False), [g_ties, eos_max(range(1, K))], n_calls=2))

    # the ends of the CDF: row 0 draws u within 2^-20 of 0 or 1 (first / last kept id); id 0 is live with p = 0 there
    def ends(rng, r):
        if r:
            return dy(rng, r)
        ids = np.array(sorted({1, 33, SLOT + 1 if V > SLOT + 1 else 40, V - 9, V - 1}))
        row = mass_row(V, ids, [0.2, 0.1, 0.3, 0.15, 0.25], np.float32(-1e4))
        row[0] = -1e4
        return row

    for nm, seed in (("cdf_low", SEED_LOW), ("cdf_high", SEED_HIGH)):
        out.append(_designed(V, nm, rng, gen(seed=seed, row_base=ENDS_ROW_BASE), [ends], n_calls=1))
    # the last_nz fallback: u = 1 - 2^-23 and row 0's scan total rounds below u * s (test_fallback_row_rounds_the_scan_below_u_s)
    fb = _designed(V, "cdf_fallback", rng, gen(seed=SEED_TOP, row_base=ENDS_ROW_BASE),
                   [lambda rng, r: fallback_row(V) if r == 0 else dy(rng, r)], n_calls=1)
    fb["calls"][0]["fallback"] = {0: FALLBACK_IDS[-1]}
    out.append(fb)

    if ext:
        def ext_gen(**kw):
            return gen(ext={**EXT_OFF, **kw})

        out.append(_designed(V, "min_p", rng, ext_gen(min_p=0.1), [mrow(MINP_ROW), mrow(MAXTIE), straddle(), flat]))
        out.append(_designed(V, "typical", rng, ext_gen(typical_p=0.7), [mrow(MAXTIE), mrow(PEAK2), straddle(), flat]))
        out.append(_designed(V, "epsilon", rng, ext_gen(epsilon_cutoff=0.025), [straddle(), mrow(MAXTIE), mrow(TAIL), flat]))
        out.append(_designed(V, "eta", rng, ext_gen(eta_cutoff=0.012), [straddle(), mrow(PEAK2), mrow(TAIL), flat]))
        out.append(_designed(V, "ext_all", rng, gen(temperature=0.8, top_k=9, top_p=0.9, ext={**EXT_OFF, "min_p": 0.02,
                             "typical_p": 0.95, "epsilon_cutoff": 3e-4, "eta_cutoff": 3e-4}), [straddle(0.8), mrow(PEAK2, 0.8)]))
        # n-gram bans on ids of the last slot: the history a_r, x_r, a_r (forced) bans x_r, which then holds the max
        last = (V - 1) // SLOT * SLOT
        xs = np.array([V - 1 - (3 * r) % (V - last) for r in range(R)])
        assert xs.min() >= last and EOS not in xs
        a = np.array([2 + r for r in range(R)])
        forced = [a, xs, a, None]

        def ngram_row(rng, r):
            row = rng.standard_normal(V).astype(np.float32)
            row[EOS] = NEG
            row[xs[r]] = 9.0
            row[[i for i in pick_ids(rng, V, 8) if i != xs[r]][:3]] = [8.0, 7.5, 7.0]
            return row

        out.append(_designed(V, "ngram_last_slot", rng, ext_gen(no_repeat_ngram_size=2), [ngram_row], n_calls=4, forced=forced))
    return [settle(grp, V) for grp in out]


SEED_CANDIDATES = [(2 ** 64 - 1 - i * 0x9E3779B97F4A7C15) % 2 ** 64 for i in range(64)]


def settle(group, V: int):
    """Designed groups draw with the first 64-bit seed (2^64 - 1 first) whose draws all stay clear of a boundary; row_base is
    nonzero.  Groups with a seed of their own keep it."""
    g = group["gen"]
    if g["seed"] in (SEED_LOW, SEED_HIGH, SEED_HIT, SEED_TOP) or not g["do_sample"]:
        return group
    g["row_base"] = 4096 + V
    for s in SEED_CANDIDATES:
        g["seed"] = s
        res = simulate(group, V)
        if not any(r["band"].any() for r, c in zip(res, group["calls"]) if c["forced"] is None and not c["exact"]):
            return group
    raise AssertionError(f"no seed keeps the draws of {group['name']} (V = {V}) clear of a boundary")


_GROUP_CACHE: dict = {}


def groups_for(V: int):
    if V not in _GROUP_CACHE:
        _GROUP_CACHE[V] = design_groups(V)
    return _GROUP_CACHE[V]


# ---- host tests --------------------------------------------------------------------------------------------------------------
def test_philox_known_answers():
    kat = [([0, 0, 0, 0], [0, 0], [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]),
           ([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2, [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]),
           ([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0],
            [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1])]
    for ctr, key, want in kat:
        assert [int(c) for c in philox4x32_10(ctr, key)] == want
    # vectorised == one at a time; the key's high word and the counter's order matter
    rows, cols = np.array([0, 1, 7, 2 ** 31 - 1]), np.array([1, 1, 2580, 3])
    u = philox_uniform(2 ** 64 - 1, rows, cols)
    assert all(u[i] == philox_uniform(2 ** 64 - 1, rows[i], cols[i]) for i in range(4))
    assert ((0 <= u) & (u < 1)).all() and (u * 2 ** 24 == np.round(u * 2 ** 24)).all()
    assert (u != philox_uniform(2 ** 32 - 1, rows, cols)).all() and (u != philox_uniform(2 ** 64 - 1, cols, rows)).any()


def test_special_seeds_put_u_where_the_cases_need_it():
    assert philox_uniform(SEED_LOW, ENDS_ROW_BASE, 1) < 2.0 ** -20
    assert philox_uniform(SEED_HIGH, ENDS_ROW_BASE, 1) > 1 - 2.0 ** -20
    hit = philox_uniform(SEED_HIT, ENDS_ROW_BASE, 1) * 64
    assert hit == 60.0
    assert philox_uniform(SEED_TOP, ENDS_ROW_BASE, 1) == 1 - 2.0 ** -23


def test_fallback_row_rounds_the_scan_below_u_s():
    """Row 0 of cdf_fallback in the kernel's float32 order.  The CTA sum (warp_sum: xor butterfly over 16, 8, 4, 2, 1, then the
    warps in order) adds lanes 1 and 17 first and rounds 1 + 2 e^-17 up to 1 + 2^-23; the inverse-CDF scan (shfl_up over 1, 2,
    4, 8, 16) adds each small mass to 1 on its own and stays at 1.  u * s then rounds to 1, no cumulative sum exceeds it, and
    the kernel takes its last id with p > 0 (last_nz).  The float64 draw is another id: the row sits in the rounding band."""
    b = np.float32(np.exp(np.float32(-17.0)))
    assert b < 0.75 * 2.0 ** -24 and 2 * b > 1.25 * 2.0 ** -24   # the same outcome for any expf within a few ulps
    e = np.zeros(32, np.float32)
    e[[i - 32 for i in FALLBACK_IDS]] = [1.0, b, b]
    lanes = np.arange(32)
    v = e.copy()
    for o in (16, 8, 4, 2, 1):
        v = (v + v[lanes ^ o]).astype(np.float32)
    x = e.copy()
    for o in (1, 2, 4, 8, 16):
        y = np.concatenate([np.zeros(o, np.float32), x[:-o]])
        x = np.where(lanes >= o, x + y, x).astype(np.float32)
    s = v[0]
    target = np.float32(np.float32(philox_uniform(SEED_TOP, ENDS_ROW_BASE, 1)) * s)
    assert s == np.float32(1 + 2.0 ** -23) and x[-1] == 1 and target == 1
    assert not (x > target).any()
    for V in (96, 2304):
        r = simulate(next(g for g in groups_for(V) if g["name"] == "cdf_fallback"), V)[0]
        assert r["band"][0] and r["drawn"][0] != FALLBACK_IDS[-1]


def _tie_free_rows(rng, R, V):
    return (rng.standard_normal((R, V)) * 2).astype(np.float32)


@pytest.mark.parametrize("knobs", [dict(top_k=7), dict(top_p=0.8), dict(temperature=0.6, top_k=40, top_p=0.9),
                                   dict(temperature=2.0, top_p=0.3), dict(do_sample=False)], ids=str)
def test_reference_equals_pinned_oracle_on_tie_free_rows(knobs):
    """Tie-free rows: the reference's processed scores equal oracle/sampling.py's (pinned to transformers), bit for bit, and
    greedy is np.argmax."""
    rng = np.random.default_rng(3)
    R, V = 12, 1088
    x = _tie_free_rows(rng, R, V)
    g = gen(**knobs)
    parler = ParlerLogitsProcessorOracle(1024, 4, 3)
    hist = np.full((R, 1), 1025, np.int64)
    g["eos"] = 1024
    res = reference_call(x, hist, g, parler, np.ones(R, bool), 1)
    want = osamp.process_scores(x, hist, ParlerLogitsProcessorOracle(1024, 4, 3), dict(g))
    assert np.array_equal(res["scores"], want)
    if not g["do_sample"]:
        assert np.array_equal(res["drawn"], want.argmax(-1))


@pytest.mark.parametrize("knobs", [dict(min_p=0.05), dict(typical_p=0.8), dict(epsilon_cutoff=3e-4), dict(eta_cutoff=1e-3)],
                         ids=str)
def test_reference_ext_equals_pinned_oracle_on_tie_free_rows(knobs):
    """The EXT warpers of the reference keep what tests/sampling_ext_oracle.py (pinned to transformers) keeps."""
    rng = np.random.default_rng(4)
    R, V = 12, 1088
    x = _tie_free_rows(rng, R, V)
    g = gen(top_p=0.97, ext={**EXT_OFF, **knobs}, eos=1024)
    hist = np.full((R, 1), 1025, np.int64)
    res = reference_call(x, hist, g, ParlerLogitsProcessorOracle(1024, 4, 3), np.ones(R, bool), 1, tol=1e-5)
    want = so.process_scores(x, hist, ParlerLogitsProcessorOracle(1024, 4, 3), dict(g, **knobs))
    diff = np.isfinite(res["scores"]) != np.isfinite(want)
    assert not (diff & ~res["near"]).any(), int(diff.sum())
    both = np.isfinite(want) & np.isfinite(res["scores"])
    assert np.array_equal(res["scores"][both], want[both])


def test_reference_group_rule_keeps_a_superset_of_transformers_on_ties():
    """bf16-rounded rows are full of ties: the group rule keeps every id transformers keeps; the extra ids lie in the one tie
    group at the threshold or in the group tied at the max."""
    rng = np.random.default_rng(5)
    R, V = 64, 1088
    x = torch.from_numpy(rng.standard_normal((R, V)).astype(np.float32) * 1.5).bfloat16().float().numpy()
    extra_rows = 0
    for top_p in (0.5, 0.8, 0.95):
        g = gen(top_p=top_p, eos=1024)
        got = np.stack([sample_row(x[r], np.zeros(V, bool), g, 0.5)[0] for r in range(R)])
        want = osamp.top_p(x.copy(), top_p)   # torch.sort ascending; ties in sort order
        kg, kw = np.isfinite(got), np.isfinite(want)
        assert not (kw & ~kg).any()
        for r in np.nonzero((kg != kw).any(1))[0]:
            vals = np.unique(x[r][kg[r] & ~kw[r]])
            assert vals.size == 1, vals
            thr = x[r][kg[r]].min()
            assert vals[0] == thr or vals[0] == x[r].max()
            extra_rows += 1
    assert extra_rows > 0, "the rows should have tie groups at the threshold"


@pytest.mark.parametrize("V", VOCABS)
def test_designed_cases_are_clear_of_every_threshold(V):
    """Designed rows: no threshold quantity within 1e-3 of its threshold and no draw within 1e-5 * S of a boundary (dyadic rows
    are exact and exempt), so the GPU checks on them can be exact."""
    for grp in groups_for(V):
        res = simulate(grp, V, tol=TOL_DESIGN)
        for i, (r, c) in enumerate(zip(res, grp["calls"])):
            assert not r["near"].any(), (grp["name"], i, np.argwhere(r["near"])[:4])
            if not c["exact"] and c["forced"] is None:
                band = r["band"].copy()
                band[list(c.get("fallback", {}))] = False   # in the band by construction
                assert not band.any(), (grp["name"], i, np.nonzero(band)[0])
            kept = np.isfinite(r["scores"]).sum(1)
            assert (kept >= 1).all()


def test_dyadic_case_draws_floor_u_n():
    V = 2304
    grp = next(g for g in groups_for(V) if g["name"] == "dyadic")
    for r, c in zip(simulate(grp, V), grp["calls"]):
        for i in range(B * K):
            live = np.nonzero(c["rows"][i] == c["rows"][i].max())[0]
            assert r["drawn"][i] == live[int(math.floor(r["u"][i] * live.size))]


@pytest.mark.parametrize("V", VOCABS)
def test_planted_case_sees_the_modelled_kernel_bugs(V):
    """Each modelled kernel bug changes the expected scores or token of at least one designed case at this vocabulary size."""
    groups = groups_for(V)
    base = [simulate(g, V) for g in groups]
    missed = []
    for bug in BUGS:
        if bug in MULTI_SLOT_BUGS and V <= SLOT:
            continue
        seen = False
        for g, ref in zip(groups, base):
            for a, b in zip(ref, simulate(g, V, bug)):
                if not np.array_equal(a["scores"], b["scores"]) or not np.array_equal(a["token"], b["token"]):
                    seen = True
                    break
            if seen:
                break
        if not seen:
            missed.append(bug)
    assert not missed, f"V = {V}: no designed case sees {missed}"


def test_reference_sees_bug():
    """The draw's sensitivity in one line each: the carry and the order at a multi-slot vocabulary, > against >= on an exact
    boundary, the ends of the CDF."""
    V = 1088
    groups = {g["name"]: g for g in groups_for(V)}
    ref = simulate(groups["dyadic_boundary"], V)[0]
    alt = simulate(groups["dyadic_boundary"], V, "ge")[0]
    live = np.nonzero(groups["dyadic_boundary"]["calls"][0]["rows"][0] == 2.5)[0]
    assert ref["drawn"][0] == live[60] and alt["drawn"][0] == live[59]
    low = simulate(groups["cdf_low"], V)[0]["drawn"][0]
    high = simulate(groups["cdf_high"], V)[0]["drawn"][0]
    assert (low, high) == (1, V - 1)
    dy = groups["dyadic"]
    assert any((simulate(dy, V)[i]["drawn"] != simulate(dy, V, "carry")[i]["drawn"]).any() for i in range(3))


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
def _tiny_model(V: int):
    from oracle.weights import make_dac_weights, make_decoder_weights
    from oracle.config import tiny_dac_cfg
    from tests.helpers import build_product_model
    cfg = tiny_cfg(vocab_size=V)
    w = make_decoder_weights(cfg, seed=3)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=min(cfg.codebook_size, V - 8))
    return cfg, build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.float32)


MAX_LEN = 24


def _begin(sess, g, inputs):
    enc, prompt = inputs
    ext = g["ext"]
    sess.begin(MAX_LEN, do_sample=g["do_sample"], temperature=g["temperature"], top_k=g["top_k"], top_p=g["top_p"],
               min_new_tokens=g["min_new_tokens"], seed=g["seed"], suppress_special=g["suppress_special"],
               codebook_size=g["codebook_size"], row_base=g["row_base"], ext=ext)
    sess.prefill(prompt, None, enc, None)


def _sample_phase(sess, n_ctas: int):
    from parler_tts_b200 import _lib
    _lib.check(_lib.lib().ptts_op_sample_phase(sess.h, int(n_ctas), _lib.stream_ptr()))


def _read(sess, cur):
    torch.cuda.synchronize()
    return sess.scores.cpu().numpy().copy(), sess.raw_ids[:, cur].cpu().numpy().copy()


# rows B*K = 12: R = 1 with as many CTAs as rows and with more; full three-row passes (4); a second loop iteration (3); three-row
# passes with invalid rows (11, 5)
PHASE_CTAS = (12, 40, 4, 3, 11, 5)


def _run_designed(V: int, phase: bool):
    cfg, model = _tiny_model(V)
    R = B * K
    P, S = 2, 4
    sess = model.decoder.engine.session(B, P, S, P + MAX_LEN)
    g0 = torch.Generator().manual_seed(1)
    inputs = (torch.randn(B, S, cfg.hidden_size, generator=g0).to(DEV), torch.randn(B, P, cfg.hidden_size, generator=g0).to(DEV))
    exact = band_free = exempt = fallbacks = phase_calls = 0
    for grp in groups_for(V):
        g = grp["gen"]
        if phase and g["ext"] is not None:
            continue
        _begin(sess, g, inputs)
        for cur, (call, ref) in enumerate(zip(grp["calls"], simulate(grp, V)), start=1):
            where = f"V={V} {grp['name']} call {cur}"
            sess.logits.copy_(torch.from_numpy(call["rows"]).to(DEV))
            fallback = call.get("fallback", {})
            want = ref["token"].copy()
            want[list(fallback)] = list(fallback.values())   # the kernel's last-id fallback on a row built to reach it

            def poison():   # every launch must write every row: nothing left over from the launch before can pass
                sess.scores.fill_(float("nan"))
                sess.raw_ids[:, cur].fill_(-1)

            if phase:
                outs = []
                for n in PHASE_CTAS:
                    poison()
                    _sample_phase(sess, n)
                    outs.append(_read(sess, cur))
                    assert int(sess.state[0].item()) == cur, "the hook must leave cur_len alone"
                    phase_calls += 1
            forced = None if call["forced"] is None else torch.from_numpy(call["forced"])
            poison()
            sess.sample(forced)
            scores, tok = _read(sess, cur)
            assert int(sess.state[0].item()) == cur + 1
            # kept set and values: bitwise, -inf where removed
            bad = np.argwhere(~((scores == ref["scores"]) | (np.isneginf(scores) & np.isneginf(ref["scores"]))))
            assert bad.size == 0, (where, bad[:5], scores[tuple(bad[0])], ref["scores"][tuple(bad[0])])
            assert np.array_equal(tok, want), (where, tok, want, ref["u"])
            if call["forced"] is None and g["do_sample"]:
                if call["exact"]:
                    exact += R
                else:
                    band_free += R - len(fallback)
                    fallbacks += len(fallback)
                    exempt += int(ref["band"].sum()) - len(fallback)
            if phase:
                for n, (s2, t2) in zip(PHASE_CTAS, outs):
                    assert np.array_equal(s2.view(np.uint32), scores.view(np.uint32)), (where, n)
                    assert np.array_equal(t2, tok), (where, n, t2, tok)
    return exact, band_free, exempt, fallbacks, phase_calls


@pytest.mark.gpu
@pytest.mark.parametrize("V", VOCABS)
def test_sampler_matches_reference(V):
    """ptts_sample (plain and EXT kernels) on the designed rows: scores bit for bit, every token the reference's."""
    exact, band_free, exempt, fallbacks, _ = _run_designed(V, phase=False)
    print(f"\nV={V}: {exact} dyadic draws exact, {band_free} other draws equal to the float64 inverse CDF, "
          f"{exempt} band exemptions, {fallbacks} last-id fallback")
    assert exempt == 0


@pytest.mark.gpu
@pytest.mark.parametrize("V", (96, 1088, 1288, 2304))
def test_sample_phase_matches_ptts_sample(V):
    """ptts_op_sample_phase (the step kernels' passes of up to three rows) with every grid shape of PHASE_CTAS: the scores and
    tokens of ptts_sample, bit for bit, on every non-EXT designed call."""
    *_, n = _run_designed(V, phase=True)
    assert n > 0


@pytest.mark.gpu
def test_vocab_above_2304_and_ext_are_refused():
    from parler_tts_b200 import _lib
    cfg, model = _tiny_model(2312)
    sess = model.decoder.engine.session(1, 2, 4, 2 + MAX_LEN)
    inputs = (torch.randn(1, 4, cfg.hidden_size).to(DEV), torch.randn(1, 2, cfg.hidden_size).to(DEV))
    _begin(sess, gen(), inputs)
    with pytest.raises(ValueError, match="2304"):
        sess.sample()
    with pytest.raises(ValueError, match="2304"):
        _sample_phase(sess, 4)
    cfg, model = _tiny_model(96)
    sess = model.decoder.engine.session(1, 2, 4, 2 + MAX_LEN)
    inputs = (torch.randn(1, 4, cfg.hidden_size).to(DEV), torch.randn(1, 2, cfg.hidden_size).to(DEV))
    _begin(sess, gen(ext={**EXT_OFF, "min_p": 0.1}), inputs)
    with pytest.raises(ValueError, match="sampling_ext"):
        _sample_phase(sess, 4)
    _begin(sess, gen(), inputs)
    sess.set_outputs(None, torch.zeros(4 * 96, device=DEV), 0, 1, 4 * 96)
    with pytest.raises(ValueError, match="sampling_ext"):
        _sample_phase(sess, 4)
    with pytest.raises(ValueError, match="n_ctas"):
        sess.set_outputs(None, None)
        _sample_phase(sess, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("knobs", [dict(top_p=0.8), dict(temperature=0.8, top_k=50, top_p=0.95)], ids=["topp0.8", "t0.8-k50-p0.95"])
def test_realistic_bf16_rows_meet_the_group_rule(knobs):
    """A bf16 Mini-shaped model (2 layers): its logits are bf16-rounded, so rows are full of ties.  The kept set equals the
    group-rule reference except where a cumulative sum lies within 1e-6 * S of a threshold; kept values are bitwise; each draw
    is the float64 inverse CDF's unless u * S lies within 1e-5 * S of a boundary.  Prints how many rows transformers' sorted-
    position rule would cut differently."""
    from oracle.weights import make_dac_weights, make_decoder_weights
    from oracle.config import tiny_dac_cfg
    from tests.helpers import build_product_model, synth_inputs
    cfg = mini_cfg(num_hidden_layers=2)
    w = make_decoder_weights(cfg, seed=21, head_std=0.3)
    dcfg = tiny_dac_cfg(n_codebooks=cfg.num_codebooks, codebook_size=cfg.codebook_size)
    model = build_product_model(cfg, dcfg, w, make_dac_weights(dcfg, seed=1), dtype=torch.bfloat16)
    Bm, Sm, Pm, L = 2, 8, 4, 16
    enc, enc_mask, prompt, prompt_mask = synth_inputs(cfg, Bm, Sm, Pm, seed=5)
    g = gen(eos=cfg.eos_token_id, pad=cfg.pad_token_id, seed=2 ** 64 - 1, row_base=9 * 7, **knobs)
    sess = model.decoder.engine.session(Bm, Pm, Sm, Pm + L)
    sess.begin(L, do_sample=True, temperature=g["temperature"], top_k=g["top_k"], top_p=g["top_p"], seed=g["seed"],
               row_base=g["row_base"])
    sess.prefill(prompt.to(DEV).bfloat16(), prompt_mask, enc.to(DEV).bfloat16(), enc_mask)
    K9 = cfg.num_codebooks
    parler = ParlerLogitsProcessorOracle(cfg.eos_token_id, K9, Bm)
    flips = band = rows = hf_rows = ties = 0
    for cur in range(1, L - 1):
        if cur > 1:
            sess.decode_forward()
        logits = sess.logits.cpu().numpy().copy()
        hist = sess.raw_ids[:, :cur].cpu().numpy()
        unf = ~(hist[:, 1:] == cfg.eos_token_id).any(1)
        ref = reference_call(logits, hist, g, parler, unf, cur)
        mask, _ = mask_matrix(hist, g, parler, logits.shape[1])
        parler = ref["parler"]
        sess.sample()
        scores, tok = _read(sess, cur)
        kd, kr = np.isfinite(scores), np.isfinite(ref["scores"])
        assert not ((kd != kr) & ~ref["near"]).any(), cur
        flips += int((kd != kr).sum())
        both = kd & kr
        assert np.array_equal(scores[both].view(np.uint32), ref["scores"][both].view(np.uint32))
        same = tok == ref["token"]
        assert (same | (ref["band"] & unf)).all(), (cur, tok, ref["token"])
        band += int((~same).sum())
        rows += tok.size
        # transformers' rule on the same scores before top-p
        pre = gen(**{**g, "top_p": 1.0})
        before = np.stack([sample_row(logits[r], mask[r], pre, 0.5)[0] for r in range(tok.size)])
        ties += int(sum(np.unique(r[np.isfinite(r)]).size < np.isfinite(r).sum() for r in before))
        if g["top_p"] < 1.0:
            hf = osamp.top_p(before.copy(), g["top_p"])
            hf_rows += int((np.isfinite(hf) != kr).any(1).sum())
    print(f"\n{knobs}: {rows} rows ({ties} with tied scores), {flips} kept-set flips at a threshold, {band} draws in the 1e-5 band, "
          f"{hf_rows} rows where transformers' sorted-position top-p keeps a different set")
