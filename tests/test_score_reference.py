"""The teacher-forced scoring kernels on their own, against a float64 reference, through the ptts_op_score hook.

Kernels (score.cu): path 1 is the fused route of ptts_score: gather_label_rows_kernel (label row b*T + t is row P + t of
utterance b, copied into xs with its two-pass LayerNorm mean / rstd), then ce_fused_kernel (the wgmma pipeline of the prefill
GEMM over the row-major folded heads: 128-row tiles, n-tiles of 128 vocabulary columns, a 3-stage TMA ring of 64-wide K stages
that runs on across n-tiles, and an epilogue that rounds each logit to bf16 and keeps a running max / sum of exp2 per row).
Path 0 is the unfused route: the decoder's heads GEMM (launch_linear, f32 logits) over the B rows of one frame, then
score_rows_kernel.  ce_reduce_kernel sums and counts the NLL per codebook on both.  ptts_score calls the same launch sequence.

Reference.  Per label row, the logits from the values the kernel sees, in float64: the LayerNorm with the true statistics (fp32
gamma / beta) and the heads as packed, in the folded form the blob holds, z = r sum_k (x_k - mu) W'_k + sum_k beta_k W_k with
W' = bf16(gamma W) recomputed on the host (test_linear_reference.linear_f64 with folded=True).  That is LN(x) W^T moved by
exactly the linear test's E_fold, so the fold's one rounding is reproduced rather than bounded: a bound of E_fold would leave about
half of all logits with two bf16 candidates, and the NLL interval a few 1e-2 nats wide.  The bound E is the linear test's E_acc +
E_ln (E_acc's chain: H/16 wgmma k-steps + 32) plus 2 u |z| for float64 -> fp32.  The kernel's bf16 logit of column c lies in
{rn(z_c - E), rn(z_c + E)} = {lo_c, hi_c}.  NLL = lse(l) - l_y grows with every l_c, c != y, and falls with
l_y (d/dl_y = p_y - 1 <= 0), so two float64 evaluations bound every NLL those logits allow:
  NLL_lo = lse(lo with hi at y) - hi_y,  NLL_hi = lse(hi with lo at y) - lo_y  (usually lo = hi and the interval is a point).

E_ce, the fp32 error of the fused kernel's log-sum-exp on exact bf16 logits (u = 2^-24; nats):
  argument  t_c = fl(l_c * fl(log2 e)): 2 u |t_c| (the constant and the product), i.e. 2 u max|l| in nats on each term, and the
            subtraction t_c - m: u |l_c - m| <= u range                                          -> 2 u max|l| + u range
  exp2f     2 ulp: 4 u relative                                                                   -> 4 u
  sums      all terms positive, so a chain's rounding is relative to the sum: 32 columns per thread and n-tile (31 u of the
            tile sum; 32 u of s over the tiles), per n-tile the rescale of the running sum (exp2f 4 u, its argument u |dm| ln 2,
            the product u, the add u: 6 u per tile, the |dm| summing to at most the range), and the quad combine (two rounds
            of two exp2f, two products, one add and their arguments: 14 u + 2 u range)           -> 46 u + 6 u n_tiles + 3 u range
  log2f     1 ulp of log2 s, s <= V                                                                -> 2 u (ln V + 1)
  (m + log2 s) ln 2: the add and the product with an fp32 ln 2                                    -> 3 u |lse|
  lse - l_y the final subtraction                                                                 -> u (|lse| + |l_y|)
  E_ce = u (2 max|l| + 4 range + 6 n_tiles + 52 + 2 ln V + 4 |lse| + |l_y|): a few 1e-5 nats for logits of tens at V = 8192,
  ~1e-5 at Mini.  The fused NLL must lie in [NLL_lo - E_ce, NLL_hi + E_ce].

Path 0 is checked in two pieces.  Its logits out_logits[b*K + k][t] must be bit-identical to ptts_op_linear2 on the lm heads
(tensor 20, f32 epilogue, path 0) over the same B rows of frame t; test_linear_reference holds those to float64.  Its NLL must
match the float64 log-softmax of those returned logits within E_rows, score_rows_kernel's fp32 error: the max is exact; expf of
l_c - m (the subtraction u range, 2 ulp = 4 u), a sum of ceil(V/256) terms per thread, 5 warp levels and 8 warp partials
(u (ceil(V/256) + 13)), logf (2 u (ln V + 1)), m + log s (u |lse|) and the final subtraction (u (|lse| + |l_y|)):
  E_rows = u (range + ceil(V/256) + 19 + 2 ln V + 2 |lse| + |l_y|).

gather_label_rows_kernel: xs must be the label rows bit for bit (never a prompt row), and (mean, rstd) must match float64
within the bound that the linear test's E_ln assumes for row statistics, 4 u (H/32 + 16) relative on rstd and of mean|x| on the
mean.  ce_reduce_kernel: the count is exact; the sum is fp32 of the float64 sum of the kernel's own counted NLL within one fp32 ulp
(it adds in double).  A cell that does not count (modeling.scoring_label_mask: label -100, a BOS label, or decoder input eos) must
be exactly 0.  Every output starts as NaN with NaN entries past its shape: everything inside must be written, nothing past it.
The same call twice gives the same bits.

Inputs are chosen to see bugs: the linear test's weights (head rows with x40 outliers, gamma log-uniform over [0.05, 20], beta of
order 1) and residual rows (mean offsets, four features 50-100x the rest, an all-zero and a constant row); label columns at
0, 7, 8, 127, 128, 1023, 1024, V - 1, eos / pad; rows steered towards one head row at those columns so that it dominates (p up
to ~1), labelled with the dominant column (NLL ~ 0: cancellation) or the least likely one; an all-equal row (zero beta, zero
row: NLL = ln V exactly); decoder-input eos cells at random, so that reading dec_ids in the labels' [B][T][K] layout masks other
cells.  The host tests check that each modelled kernel bug moves the reference past 4x the bar on some cell of its case.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import math

import pytest
import torch

from oracle.config import decoder_cfg
from parler_tts_b200.modeling import scoring_label_mask
from tests.test_linear_reference import MATRICES, U, bf16, engine, linear_f64, make_layer, make_weights, residual_rows

DEV = "cuda"
NT = 128                         # vocabulary columns per n-tile of ce_fused_kernel
EDGE_COLS = (0, 7, 8, 127, 128, 1023, 1024)
# (H, V, K): 1, 2 and 3 K stages against the 3-stage ring, Mini and Large widths; one partial tile, exact tiles, half and odd
# partial last tiles and the fused kernel's limit V = 8192 (c1 / c2 take 64 KB of shared memory there)
CASES = [(64, 1088, 9), (128, 1088, 9), (192, 1088, 9), (1024, 1088, 9), (1536, 1088, 9),
         (128, 8, 9), (64, 64, 9), (192, 120, 9), (128, 128, 2), (64, 136, 9), (1024, 1024, 2), (128, 1096, 2),
         (192, 2048, 2), (64, 8192, 1), (128, 8192, 2), (1536, 8192, 1)]
F32_CASES = [(128, 1088, 9), (64, 136, 9), (128, 8, 9), (1024, 8192, 1)]
# (B, T, P): B*T = 1, 127, 128, 129, 255, 256, 257 label rows
ROWS = [(1, 1, 0), (1, 127, 1), (2, 64, 32), (3, 43, 0), (5, 51, 1), (4, 64, 32), (1, 257, 1)]
ZERO_BETA = {(128, 1088, 9), (64, 8192, 1)}   # cases with beta = 0: their all-zero rows have all-equal logits
WORST: dict = {}                 # (path, dtype, H, V) -> worst error / bar (fused: distance outside [NLL_lo, NLL_hi] / E_ce)


def score_cfg(H, V, K):
    eos, bos = (1024, 1025) if V >= 1024 else (V // 2, V // 2 + 1)
    return decoder_cfg(hidden_size=H, num_attention_heads=H // 64, ffn_dim=H, vocab_size=V, num_codebooks=K, num_hidden_layers=1,
                       max_position_embeddings=16, pad_token_id=eos, eos_token_id=eos, bos_token_id=bos)


def score_weights(cfg):
    """The linear test's weights with the head rows at the edge columns 3x the rest, so that a row steered towards one of them
    is dominated by it (with 0.02 N(0, 1) heads and gamma log-uniform over [0.05, 20] no column reaches p = 0.5 at small H)."""
    w = make_weights(cfg, seed=11)
    for k in range(cfg.num_codebooks):
        w[f"decoder.lm_heads.{k}.weight"][edge_columns(cfg)] *= 3.0
    if (cfg.hidden_size, cfg.vocab_size, cfg.num_codebooks) in ZERO_BETA:
        w["decoder.model.decoder.layer_norm.bias"].zero_()
    return w


# ---- the reference ------------------------------------------------------------------------------------------------------
def logits_f64(layer, xr, V):
    """z [R, K, V] in float64 and the bound E on the kernel's fp32 value before its bf16 rounding (incl. float64 -> fp32)."""
    y, E = linear_f64(layer, xr, folded=True)
    E = E + 2 * U * y.abs()
    return y.view(len(y), -1, V), E.view(len(y), -1, V)


def lse(l):
    return torch.logsumexp(l, -1)


def e_ce(lo, hi, ly, V):
    m = hi.amax(-1)
    amax = torch.maximum(lo.abs(), hi.abs()).amax(-1)
    rng = m - lo.amin(-1)
    s = lse(hi).abs()
    return U * (2 * amax + 4 * rng + 6 * math.ceil(V / NT) + 52 + 2 * math.log(V) + 4 * s + ly.abs())


def e_rows(l, ly, V):
    rng = l.amax(-1) - l.amin(-1)
    s = lse(l).abs()
    return U * (rng + math.ceil(V / 256) + 19 + 2 * math.log(V) + 2 * s + ly.abs())


def nll_interval(z, E, lab):
    """(NLL_lo, NLL_hi, E_ce) [R, K] for labels lab [R, K] (any column; masked cells too)."""
    lo, hi = bf16(z - E), bf16(z + E)
    idx = lab.clamp(min=0).unsqueeze(-1)
    hy, ly = hi.gather(-1, idx), lo.gather(-1, idx)
    n_lo = lse(lo.scatter(-1, idx, hy)) - hy[..., 0]
    n_hi = lse(hi.scatter(-1, idx, ly)) - ly[..., 0]
    return n_lo, n_hi, e_ce(lo, hi, ly[..., 0], z.shape[-1])


def ratios(got, mask, n_lo, n_hi, e):
    """On counted cells, how far got lies outside [NLL_lo, NLL_hi] in units of E_ce (<= 1: inside the bar); a cell that does not
    count must be exactly 0 (inf otherwise)."""
    r = ((got - (n_lo + n_hi) / 2).abs() - (n_hi - n_lo) / 2).clamp(min=0) / e
    r = torch.where(mask, r, torch.where(got == 0, torch.zeros_like(r), torch.full_like(r, math.inf)))
    return torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)


def on(layer, device):
    return dataclasses.replace(layer, W=layer.W.to(device), gamma=layer.gamma.to(device), beta=layer.beta.to(device))


# ---- cases --------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Case:
    cfg: object
    layer: object
    B: int
    P: int
    T: int
    x: torch.Tensor        # [B, P+T, H] model dtype (host)
    labels: torch.Tensor   # [B, T, K] int64
    dec: torch.Tensor      # [B*K, T] int64
    dominant: list         # (label row, codebook, column)

    @property
    def M(self):
        return self.B * self.T

    def label_rows(self, rows=None):
        xr = self.x[:, self.P:].reshape(self.M, -1).double()
        return xr if rows is None else xr[rows]

    def mask(self):
        """[M, K] bool: the cells that count (modeling.scoring_label_mask) and the labels with BOS as -100."""
        lab, m = scoring_label_mask(self.labels, self.dec, self.cfg.bos_token_id, self.cfg.eos_token_id)
        return lab.reshape(self.M, -1), m.reshape(self.M, -1)


def edge_columns(cfg):
    V = cfg.vocab_size
    return sorted({c for c in EDGE_COLS + (V - 1, cfg.eos_token_id, cfg.pad_token_id) if c < V and c != cfg.bos_token_id})


def make_case(cfg, w, B, P, T, seed, dtype=torch.bfloat16, device="cpu") -> Case:
    H, V, K = cfg.hidden_size, cfg.vocab_size, cfg.num_codebooks
    g = torch.Generator().manual_seed(seed)
    layer = make_layer(cfg, w, MATRICES[-1], dtype)
    M = B * T
    x = residual_rows(g, B * (P + T), H).view(B, P + T, H)
    cols = edge_columns(cfg)
    # steer some label rows towards head row (k, c): x = a v + (1 - a) s, v the standardised W_kc, s the row's own
    dominant = []
    Wg = layer.W.float()
    for i, r in enumerate(range(7, M, 3)):   # round q = i // len(cols) takes every edge column once
        q = i // len(cols)
        k, c, a = q % K, cols[i % len(cols)], (1.0, 0.6, 0.35)[q % 3]
        v = Wg[k * V + c]
        xr = x[r // T, P + r % T]
        s = (xr - xr.mean()) / xr.std().clamp(min=1e-6)
        x[r // T, P + r % T] = (a * (v - v.mean()) / v.std() + (1 - a) * s) * xr.abs().mean().clamp(min=0.5) + xr.mean()
        dominant.append((r, k, c))
    x = x.to(dtype)
    labels = torch.randint(0, V, (M, K), generator=g)
    cell = torch.arange(M * K).view(M, K)
    edge = cell % 3 == 0
    labels[edge] = torch.tensor(cols)[(cell[edge] // 3) % len(cols)]
    # the dominant rows: the dominant column (NLL ~ 0) for three rounds, then the least likely one for three
    if dominant:
        rows = torch.tensor([d[0] for d in dominant])
        z, _ = logits_f64(on(layer, device), x[:, P:].reshape(M, H)[rows].double().to(device), V)
        for j, (r, k, c) in enumerate(dominant):
            labels[r, k] = c if (j // len(cols) // 3) % 2 == 0 else int(z[j, k].argmin())
    labels[cell % 17 == 5] = -100
    if cfg.bos_token_id < V:
        labels[cell % 19 == 7] = cfg.bos_token_id
    dec = torch.randint(0, V + 1, (B * K, T), generator=g)
    dec[torch.rand(B * K, T, generator=g) < 0.1] = cfg.eos_token_id
    return Case(cfg, layer, B, P, T, x, labels.view(B, T, K), dec, dominant)


# ---- modelled kernel bugs (host) ------------------------------------------------------------------------------------------
def folded_logits(case, xr, mu, r, k_c):
    """r (x W'^T - mu c1) + c2 per codebook with c1 / c2 of codebook k_c[k] (the kernel's folded form)."""
    lay, V = case.layer, case.cfg.vocab_size
    Wf = lay.Wf
    c1 = Wf.sum(1)
    c2 = lay.beta @ lay.W.T
    K = case.cfg.num_codebooks
    out = []
    for k in range(K):
        s = slice(k * V, (k + 1) * V)
        sc = slice(k_c[k] * V, (k_c[k] + 1) * V)
        out.append(r * (xr @ Wf[s].T - mu * c1[sc][None]) + c2[sc][None])
    return torch.stack(out, 1)


def bad_nll(case, bug: str):
    """[M, K] token_nll of a kernel with bug `bug` (0 where that kernel's mask drops the cell)."""
    cfg, V, K, M = case.cfg, case.cfg.vocab_size, case.cfg.num_codebooks, case.M
    xr = case.label_rows()
    lab, mask = case.mask()
    z, _ = logits_f64(case.layer, xr, V)
    l = bf16(z)
    y = lab.clamp(min=0)
    mu = xr.mean(1, keepdim=True)
    rs = 1.0 / torch.sqrt(((xr - mu) ** 2).mean(1, keepdim=True) + case.layer.eps)

    def nll(l, y):
        return lse(l) - l.gather(-1, y.unsqueeze(-1))[..., 0]

    if bug.startswith("drop_col_"):
        c = {"tile": NT, "1024": 1024, "last": V - 1}[bug[9:]]
        keep = torch.ones(V, dtype=torch.bool)
        keep[c] = False
        out = torch.where(y == c, nll(l, y), lse(l[..., keep]) - l.gather(-1, y.unsqueeze(-1))[..., 0])
    elif bug == "tail_zero":
        assert V % NT != 0
        out = torch.logaddexp(lse(l), torch.zeros(())) - l.gather(-1, y.unsqueeze(-1))[..., 0]
    elif bug in ("label_plus1", "label_minus1", "label_pair"):
        y2 = {"label_plus1": (y + 1).clamp(max=V - 1), "label_minus1": (y - 1).clamp(min=0), "label_pair": y ^ 1}[bug]
        out = lse(l) - l.gather(-1, y2.unsqueeze(-1))[..., 0]
    elif bug in ("stats_next", "stats_prev"):
        sh = -1 if bug == "stats_next" else 1
        out = nll(bf16(folded_logits(case, xr, mu.roll(sh, 0), rs.roll(sh, 0), list(range(K)))), y)
    elif bug == "prompt_not_skipped":
        assert case.P > 0
        xw = case.x[:, :case.T].reshape(M, -1).double()
        out = nll(bf16(logits_f64(case.layer, xw, V)[0]), y)
    elif bug in ("c_next", "c_prev"):
        kc = [(k + (1 if bug == "c_next" else -1)) % K for k in range(K)]
        out = nll(bf16(folded_logits(case, xr, mu, rs, kc)), y)
    elif bug == "rescale_skip":
        # the first n-tile whose max raises the running max keeps the earlier tiles' sum unscaled
        nt = math.ceil(V / NT)
        pad = torch.full(l.shape[:-1] + (nt * NT - V,), -math.inf, dtype=l.dtype)
        tiles = torch.cat([l, pad], -1).view(*l.shape[:-1], nt, NT)
        cm = tiles.amax(-1).cummax(-1).values
        rise = torch.cat([torch.zeros_like(cm[..., :1], dtype=torch.bool), cm[..., 1:] > cm[..., :-1]], -1)
        J = torch.where(rise.any(-1), rise.float().argmax(-1), torch.full_like(cm[..., 0], nt, dtype=torch.long))
        before = torch.arange(nt) < J.unsqueeze(-1)
        tsum = torch.exp(tiles - lse(l)[..., None, None]).sum(-1)          # tile sums relative to the true total
        earlier = (tsum * before).sum(-1)
        grow = torch.exp(cm.gather(-1, J.clamp(max=nt - 1).unsqueeze(-1))[..., 0] - cm.gather(-1, (J - 1).clamp(min=0).unsqueeze(-1))[..., 0])
        grow = torch.where(J < nt, grow, torch.ones_like(grow))
        out = lse(l) + torch.log1p(earlier * (grow - 1)) - l.gather(-1, y.unsqueeze(-1))[..., 0]
    elif bug == "no_bf16_round":
        out = nll(z.float().double(), y)
    elif bug in ("eos_inverted", "bos_inverted", "dec_layout"):
        labels = case.labels.reshape(M, K)
        dec = case.dec.view(case.B, K, case.T).transpose(1, 2).reshape(M, K)
        valid = (labels != -100) & (labels != cfg.bos_token_id)
        if bug == "eos_inverted":
            mask = valid & (dec == cfg.eos_token_id)
        elif bug == "bos_inverted":
            mask = (labels != -100) & (dec != cfg.eos_token_id)
        else:
            mask = valid & (case.dec.reshape(M, K) != cfg.eos_token_id)
        out = nll(l, labels.clamp(min=0))
    else:
        raise KeyError(bug)
    return torch.where(mask, out, torch.zeros_like(out))


def host_reference(case):
    lab, mask = case.mask()
    z, E = logits_f64(case.layer, case.label_rows(), case.cfg.vocab_size)
    return (mask,) + nll_interval(z, E, lab)


SENSITIVITY = [   # (bug, (H, V, K), (B, T, P))
    ("drop_col_tile", (128, 1096, 2), (1, 257, 1)),
    ("drop_col_1024", (128, 1096, 2), (1, 257, 1)),
    ("drop_col_last", (128, 1096, 2), (1, 257, 1)),
    ("drop_col_tile", (128, 8192, 2), (1, 257, 1)),
    ("drop_col_1024", (128, 8192, 2), (1, 257, 1)),
    ("drop_col_last", (128, 8192, 2), (1, 257, 1)),
    ("tail_zero", (128, 1096, 2), (1, 257, 1)),
    ("tail_zero", (192, 120, 9), (3, 43, 0)),
    ("label_plus1", (128, 1088, 9), (3, 43, 0)),
    ("label_minus1", (128, 1088, 9), (3, 43, 0)),
    ("label_pair", (128, 1088, 9), (3, 43, 0)),
    ("stats_next", (128, 1088, 9), (3, 43, 0)),
    ("stats_prev", (128, 1088, 9), (3, 43, 0)),
    ("prompt_not_skipped", (128, 1088, 9), (2, 64, 32)),
    ("prompt_not_skipped", (64, 64, 9), (1, 127, 1)),
    ("c_next", (128, 1088, 9), (3, 43, 0)),
    ("c_prev", (128, 128, 2), (5, 51, 1)),
    ("rescale_skip", (128, 1088, 9), (3, 43, 0)),
    ("rescale_skip", (128, 8192, 2), (1, 257, 1)),
    ("no_bf16_round", (128, 1088, 9), (3, 43, 0)),
    ("no_bf16_round", (128, 8, 9), (1, 127, 1)),
    ("eos_inverted", (128, 1088, 9), (3, 43, 0)),
    ("bos_inverted", (128, 1088, 9), (3, 43, 0)),
    ("bos_inverted", (128, 8, 9), (1, 127, 1)),
    ("dec_layout", (128, 1088, 9), (3, 43, 0)),
    ("dec_layout", (64, 136, 9), (5, 51, 1)),
]


def case_seed(shape, rows):
    return (shape[0] * 7 + shape[1] * 13 + shape[2] * 31 + rows[0] * 3 + rows[1] * 5 + rows[2]) % 100003


@pytest.mark.parametrize("bug,shape,rows", SENSITIVITY)
def test_reference_sees_bug(bug, shape, rows):
    cfg = score_cfg(*shape)
    case = make_case(cfg, score_weights(cfg), rows[0], rows[2], rows[1], seed=case_seed(shape, rows))
    mask, n_lo, n_hi, e = host_reference(case)
    ratio = float(ratios(bad_nll(case, bug), mask, n_lo, n_hi, e).max())
    assert ratio > 4.0, f"{bug} on {shape} {rows} moves the reference by only {ratio:.2f}x the bar"


@pytest.mark.parametrize("shape,rows", [((128, 1096, 2), (1, 257, 1)), ((64, 64, 9), (1, 127, 1))])
def test_interval_contains_the_rounded_logits(shape, rows):
    """NLL_lo <= NLL(rn(z)) <= NLL_hi: the interval holds the NLL of the logits rounded from the exact z; most logits have a
    single bf16 candidate; the correct kernel model lands inside the bar everywhere."""
    cfg = score_cfg(*shape)
    case = make_case(cfg, score_weights(cfg), rows[0], rows[2], rows[1], seed=case_seed(shape, rows))
    lab, mask = case.mask()
    z, E = logits_f64(case.layer, case.label_rows(), cfg.vocab_size)
    n_lo, n_hi, e = nll_interval(z, E, lab)
    l = bf16(z)
    n = lse(l) - l.gather(-1, lab.clamp(min=0).unsqueeze(-1))[..., 0]
    assert bool((n_lo <= n).all()) and bool((n <= n_hi).all())
    assert float((bf16(z - E) == bf16(z + E)).float().mean()) > 0.9   # most logits have one candidate
    assert float(ratios(torch.where(mask, n, torch.zeros_like(n)), mask, n_lo, n_hi, e).max()) <= 1.0
    assert 1e-7 < float(e.max()) < 1e-3


@pytest.mark.parametrize("shape,rows", [((64, 1088, 9), (2, 64, 32)), ((128, 8192, 2), (1, 257, 1)), ((192, 120, 9), (3, 43, 0))])
def test_cases_reach_their_edges(shape, rows):
    """Every case has labels at each edge column, dominant rows with p >= 0.5 labelled both ways, masked cells of all three
    kinds, and eos cells where the labels' layout would read other ones."""
    cfg = score_cfg(*shape)
    case = make_case(cfg, score_weights(cfg), rows[0], rows[2], rows[1], seed=case_seed(shape, rows))
    lab, mask = case.mask()
    counted = set(lab[mask].tolist())
    assert set(edge_columns(cfg)) <= counted
    z, _ = logits_f64(case.layer, case.label_rows(), cfg.vocab_size)
    p = torch.softmax(bf16(z), -1)
    dom = [(r, k, c) for r, k, c in case.dominant if float(p[r, k, c]) >= 0.5]
    assert len(dom) >= 3, "too few dominant rows"
    assert any(lab[r, k] == c for r, k, c in dom) and any(lab[r, k] != c for r, k, c in dom)
    assert bool((case.labels == -100).any()) and bool((~mask & (lab != -100)).any())
    M, K = case.M, cfg.num_codebooks
    wrong = case.dec.reshape(M, K) == cfg.eos_token_id
    right = case.dec.view(case.B, K, case.T).transpose(1, 2).reshape(M, K) == cfg.eos_token_id
    assert bool((wrong != right).any())


def test_all_equal_row_scores_ln_v():
    """With beta = 0 an all-zero residual row has all logits 0: its NLL is ln V on every codebook."""
    cfg = score_cfg(128, 1088, 9)
    case = make_case(cfg, score_weights(cfg), 3, 0, 43, seed=1)
    lab, mask = case.mask()
    n_lo, n_hi, e = nll_interval(*logits_f64(case.layer, case.label_rows(), 1088), lab)
    assert torch.equal(n_lo[3], torch.full_like(n_lo[3], math.log(1088))) and torch.equal(n_lo[3], n_hi[3])


def test_hook_signature():
    from parler_tts_b200 import _lib
    assert len(_lib._SIGS["ptts_op_score"][1]) == 17



# ---- GPU ------------------------------------------------------------------------------------------------------------------
PAD = 64   # NaN entries past every output


def run_op(eng, case, path, logits=False, sums=True):
    from parler_tts_b200 import _lib
    cfg = case.cfg
    B, P, T, K, V, H, M = case.B, case.P, case.T, cfg.num_codebooks, cfg.vocab_size, cfg.hidden_size, case.M
    nan = float("nan")
    o = {"nll": torch.full((M * K + PAD,), nan, device=DEV),
         "logits": torch.full((B * K * T * V + PAD,), nan, device=DEV) if logits else None,
         "sums": torch.full((2 * K + PAD,), nan, device=DEV) if sums else None,
         "xs": torch.full(((M + 1) * H,), nan, dtype=torch.bfloat16, device=DEV) if path == 1 else None,
         "stats": torch.full((2 * M + PAD,), nan, device=DEV) if path == 1 else None}
    scratch = torch.empty(B * K * V, device=DEV) if path == 0 else None
    x = case.x.to(DEV).contiguous()
    lab, dec = case.labels.to(DEV).contiguous(), case.dec.to(DEV).contiguous()
    heads = eng.heads_rowmajor() if path == 1 else None
    _lib.check(_lib.lib().ptts_op_score(C.byref(eng.c), _lib.ptr(eng.blob), _lib.ptr(heads), _lib.ptr(x), B, P, T, _lib.ptr(lab),
                                        _lib.ptr(dec), path, _lib.ptr(o["nll"]), _lib.ptr(o["logits"]), _lib.ptr(o["sums"]),
                                        _lib.ptr(o["xs"]), _lib.ptr(o["stats"]), _lib.ptr(scratch), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return o


def record(tag, r, what):
    worst = float(r.max())
    WORST[tag] = max(WORST.get(tag, 0.0), worst)
    if worst > 1.0:
        i = int(r.flatten().argmax())
        raise AssertionError(f"{what}: {worst:.2f} x bar at cell {divmod(i, r.shape[-1])} ({int((r > 1).sum())} cells over)")


def check_written(o, n, key, what):
    v = o[key]
    assert not bool(torch.isnan(v[:n]).any()), f"{what}: {key} has unwritten entries"
    assert bool(torch.isnan(v[n:].float()).all()), f"{what}: {key} was written past its shape"


def check_sums(o, case, mask, what):
    K = case.cfg.num_codebooks
    nll = o["nll"][:case.M * K].view(case.M, K).double().cpu()
    s = o["sums"][:2 * K].view(K, 2).cpu()
    for k in range(K):
        assert float(s[k, 1]) == float(mask[:, k].sum()), f"{what}: codebook {k} count"
        ref = torch.tensor(float(nll[mask[:, k], k].sum()), dtype=torch.float32)
        ulp = float(torch.nextafter(ref.abs(), torch.tensor(math.inf)) - ref.abs())
        assert abs(float(s[k, 0]) - float(ref)) <= ulp, f"{what}: codebook {k} sum {float(s[k, 0])!r} vs {float(ref)!r}"


def check_fused(eng, case, rows=None, what=""):
    cfg, K, M, H = case.cfg, case.cfg.num_codebooks, case.M, case.cfg.hidden_size
    o = run_op(eng, case, 1)
    o2 = run_op(eng, case, 1)
    for key in ("nll", "sums", "xs", "stats"):
        assert torch.equal(o[key].view(torch.int32 if key != "xs" else torch.int16),
                           o2[key].view(torch.int32 if key != "xs" else torch.int16)), f"{what}: {key} differs between two runs"
    check_written(o, M * K, "nll", what)
    check_written(o, 2 * K, "sums", what)
    check_written(o, 2 * M, "stats", what)
    check_written(o, M * H, "xs", what)
    xl = case.x[:, case.P:].reshape(M, H)
    assert torch.equal(o["xs"][:M * H].view(M, H).cpu().view(torch.int16), xl.view(torch.int16)), f"{what}: xs is not the label rows"
    lab, mask = case.mask()
    check_sums(o, case, mask, what)
    rows = torch.arange(M) if rows is None else rows
    lay = on(case.layer, DEV)
    xr = xl[rows].double().to(DEV)
    z, E = logits_f64(lay, xr, cfg.vocab_size)
    n_lo, n_hi, e = nll_interval(z, E, lab[rows].to(DEV))
    got = o["nll"][:M * K].view(M, K)[rows.to(DEV)].double()
    record(("fused", "bf16", H, cfg.vocab_size), ratios(got, mask[rows].to(DEV), n_lo, n_hi, e).cpu(), f"{what} fused nll")
    # row statistics: the linear test's bound on its two-pass statistics
    st = o["stats"][:2 * M].view(M, 2)[rows.to(DEV)].double()
    mu = xr.mean(1)
    r = 1.0 / torch.sqrt(((xr - mu[:, None]) ** 2).mean(1) + lay.eps)
    b = 4 * U * (H / 32 + 16)
    rr = torch.maximum((st[:, 0] - mu).abs() / (b * xr.abs().mean(1) + 1e-30), (st[:, 1] / r - 1).abs() / b)
    record(("row_stats", "bf16", H, cfg.vocab_size), rr[:, None].cpu(), f"{what} row stats")


def check_unfused(eng, case, dtype, frames=None, rows=None, what=""):
    from parler_tts_b200 import _lib
    cfg, K, M, V, H = case.cfg, case.cfg.num_codebooks, case.M, case.cfg.vocab_size, case.cfg.hidden_size
    B, T = case.B, case.T
    o = run_op(eng, case, 0, logits=True)
    o2 = run_op(eng, case, 0, logits=True)
    for key in ("nll", "logits", "sums"):
        assert torch.equal(o[key].view(torch.int32), o2[key].view(torch.int32)), f"{what}: {key} differs between two runs"
    check_written(o, M * K, "nll", what)
    check_written(o, B * K * T * V, "logits", what)
    check_written(o, 2 * K, "sums", what)
    lab, mask = case.mask()
    check_sums(o, case, mask, what)
    logits = o["logits"][:B * K * T * V].view(B, K, T, V)
    x = case.x.to(DEV)
    for t in (range(T) if frames is None else frames):
        want = torch.full((B, K * V), float("nan"), device=DEV)
        _lib.check(_lib.lib().ptts_op_linear2(C.byref(eng.c), _lib.ptr(eng.blob), 20, 0, _lib.ptr(x[:, case.P + t].contiguous()), B, 1, 3,
                                              None, _lib.ptr(want), 0, None, _lib.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(logits[:, :, t].reshape(B, K * V).view(torch.int32), want.view(torch.int32)), \
            f"{what}: frame {t} logits differ from ptts_op_linear2"
    rows = torch.arange(M) if rows is None else rows
    rd = rows.to(DEV)
    l = logits.permute(0, 2, 1, 3).reshape(M, K, V)[rd].double()
    y = lab[rows].clamp(min=0).to(DEV)
    ly = l.gather(-1, y.unsqueeze(-1))[..., 0]
    n = lse(l) - ly
    got = o["nll"][:M * K].view(M, K)[rd].double()
    md = mask[rows].to(DEV)
    r = (got - n).abs() / e_rows(l, ly, V)
    r = torch.where(md, r, torch.where(got == 0, torch.zeros_like(r), torch.full_like(r, math.inf)))
    r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    record(("unfused", "bf16" if dtype == torch.bfloat16 else "f32", H, V), r.cpu(), f"{what} unfused nll")


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if WORST:
        print("\n[score reference] worst error / bar per (path, dtype, H, V): " +
              ", ".join(f"{p} {d} H{h} V{v} {w:.3f}" for (p, d, h, v), w in sorted(WORST.items())))


def score_engine(shape, dtype):
    cfg = score_cfg(*shape)
    return engine("score_%d_%d_%d" % shape, dtype, cfg=cfg, weights=score_weights)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", CASES, ids=lambda s: "H%d-V%d-K%d" % s)
def test_fused_and_unfused_bf16(shape):
    cfg, w, eng = score_engine(shape, torch.bfloat16)
    for rows in ROWS:
        B, T, P = rows
        case = make_case(cfg, w, B, P, T, seed=case_seed(shape, rows), device=DEV)
        what = f"H{shape[0]} V{shape[1]} K{shape[2]} B{B} T{T} P{P}"
        check_fused(eng, case, what=what)
        check_unfused(eng, case, torch.bfloat16, what=what)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", F32_CASES, ids=lambda s: "H%d-V%d-K%d" % s)
def test_unfused_f32(shape):
    cfg, w, eng = score_engine(shape, torch.float32)
    for rows in ROWS:
        B, T, P = rows
        case = make_case(cfg, w, B, P, T, seed=case_seed(shape, rows), dtype=torch.float32, device=DEV)
        check_unfused(eng, case, torch.float32, what=f"f32 H{shape[0]} V{shape[1]} K{shape[2]} B{B} T{T} P{P}")


@pytest.mark.gpu
def test_mini_scale():
    """B = 32, T = 430 (13 760 label rows, 107.5 row tiles) at the Mini shape: every row of the first tile, the rows on either
    side of every tile edge and of the last partial tile, and 256 random rows."""
    shape = (1024, 1088, 9)
    cfg, w, eng = score_engine(shape, torch.bfloat16)
    B, T, P = 32, 430, 32
    case = make_case(cfg, w, B, P, T, seed=7, device=DEV)
    M = B * T
    sel = set(range(128)) | set(range((M - 1) // 128 * 128, M))
    for m in range(128, M, 128):
        sel |= {m - 1, m}
    g = torch.Generator().manual_seed(8)
    sel |= set(torch.randint(0, M, (256,), generator=g).tolist())
    rows = torch.tensor(sorted(sel))
    check_fused(eng, case, rows=rows, what="mini B32 T430")
    frames = sorted({0, 1, T - 1} | set((rows[::37] % T).tolist()))
    check_unfused(eng, case, torch.bfloat16, frames=frames, rows=rows, what="mini B32 T430")


@pytest.mark.gpu
def test_hook_refuses_what_ptts_score_would_not_run():
    from parler_tts_b200 import _lib
    shape = (64, 136, 9)
    cfg, w, eng = score_engine(shape, torch.bfloat16)
    case = make_case(cfg, w, 2, 1, 5, seed=1)
    M, K, V, H = 10, 9, 136, 64
    x, lab, dec = case.x.to(DEV), case.labels.to(DEV), case.dec.to(DEV)
    nll, logits = torch.zeros(M * K, device=DEV), torch.zeros(2 * K * 5 * V, device=DEV)
    xs, st, scr = torch.zeros(M * H, dtype=torch.bfloat16, device=DEV), torch.zeros(2 * M, device=DEV), torch.zeros(2 * K * V, device=DEV)
    heads = eng.heads_rowmajor()

    def call(e, path, T=5, labels=lab, out=None, xs_=xs, st_=st, scr_=scr, heads_=heads, x_=x):
        return _lib.lib().ptts_op_score(C.byref(e.c), _lib.ptr(e.blob), _lib.ptr(heads_), _lib.ptr(x_), 2, 1, T, _lib.ptr(labels),
                                        _lib.ptr(dec), path, _lib.ptr(nll), _lib.ptr(out), None, _lib.ptr(xs_), _lib.ptr(st_),
                                        _lib.ptr(scr_), _lib.stream_ptr())

    assert call(eng, 1) == 0 and call(eng, 0) == 0
    torch.cuda.synchronize()
    for args, msg in [(dict(path=1, T=0), "T >= 1"), (dict(path=0, T=0), "T >= 1"), (dict(path=2), "path"),
                      (dict(path=1, labels=None, out=logits), "labels"), (dict(path=1, out=logits), "no logits"),
                      (dict(path=1, xs_=None), "xs_scratch"), (dict(path=1, st_=None), "row_stats"),
                      (dict(path=1, heads_=None), "heads_rm"), (dict(path=0, scr_=None), "logits_scratch")]:
        path = args.pop("path")
        assert call(eng, path, **args) == _lib.EINVAL, msg
        assert msg in _lib.lib().ptts_last_error().decode(), _lib.lib().ptts_last_error()
    cfg32, w32, eng32 = score_engine(shape, torch.float32)
    assert call(eng32, 1, x_=x.float()) == _lib.EINVAL and b"bf16" in _lib.lib().ptts_last_error()
    cfgb, wb, engb = score_engine((64, 8200, 1), torch.bfloat16)
    assert call(engb, 1) == _lib.EINVAL and b"outside the fused kernel" in _lib.lib().ptts_last_error()
