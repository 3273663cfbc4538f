"""The linear layers on their own, against a float64 reference, through the ptts_op_linear hook.

Kernels: path 0 is the decode GEMM of gemm.cu (linear_bf16_kernel: 32-row tiles, mma.sync, 1/2/3/4/6/8 n-tiles of 8 columns per
CTA, activation tile chunked when K > H; linear_f32_kernel for the f32 model dtype).  Path 1 is the wgmma prefill GEMM of
gemm_tc.cu (linear_tc_kernel: 128-row tiles, N tiles of 128 / 96 / 64 columns, a 3-stage TMA ring of 64-wide K stages, and
row_stats_kernel's two-pass LayerNorm statistics).  The 32-column N tile cannot be reached from a decoder shape: every decoder
N is a multiple of 64 (head_dim), so only the DAC convolutions use it.

The reference is the layer in float64 from exactly the values the kernel sees: the bf16 (f32) input rows, the weights as packed
(the state dict rounded to the model dtype) and fp32 gamma / beta.  LayerNorm is exact (biased variance, eps 1e-5), then
x_hat W^T, then the epilogue of the reference module: one bf16 rounding of the linear output, then erf-GELU / relu / silu /
tanh-GELU, or res + that, or the f32 logits of the lm heads.  For bf16, LayerNorm is folded into the weights at load
(ln_stats.cuh: y = r (sum_k x_k W'_k - mu c1) + c2, W' = bf16(gamma W)), and the bars model that arithmetic, not the reference's.

Bars, per element (u = 2^-24, one fp32 rounding):
  E_acc  = u (K/16 + 32) mass: the n u bound of n chained fp32 additions; products of bf16 are exact in fp32, the deepest
           chain is K/16 mma k-steps, plus the 8-warp reduction and the epilogue (< 32 more roundings).  mass is what those sums
           add up: sum_k |x_k W_k|, or with the fold r (sum_k |x_k W'_k| + |mu| sum_k |W'_k|) + sum_k |beta_k W_k| -- the sums
           of x W' and of c1 that cancel in r (sum x W' - mu c1), and c2's.  f32 dtype: n = K + 64 (one serial fmaf chain).
  E_fold = |r sum_k (x_k - mu)(W'_k - gamma_k W_k)|: the shift from rounding gamma W to bf16 once at load (the fold's only
           rounding the reference does not make).  W' is recomputed on the host as fold_layernorm_kernel defines it,
           bf16(fp32(gamma) * fp32(W)), not read back from the blob: a fold that computes something else is not excused.
  E_ln   = 4 u (K/32 + 16) (|y - c2| + r mean_k|x_k| |c1|): row statistics with the error of a well-conditioned fp32
           computation (chains of K/32 + 5 additions; rstd's relative error is half of var's, var's twice mean's).  The decode
           path's one-pass variance S2/K - mu^2 is not well conditioned when |mu|/sigma is large: the offset sweep measures it.
  dev    = the largest change of the epilogue when the fp32 linear output sits anywhere within E_acc + E_fold + E_ln (+ 2 u |y|
           for float64 -> fp32) of y: zero when that interval holds no bf16 rounding midpoint (both round the same way), one
           bf16 ulp of y pushed through the activation / residual otherwise.
  bf16 outputs:  |got - ref| <= dev + 2^-8 (|ref| + dev) + 2^-20 (|y_bf16| + |ref|)
           (2^-8: the final rounding to bf16, half an ulp; 2^-20: a few fp32 ulps of erff / expf / tanhf, and the absolute
           error of 1 + erf(x / sqrt 2) near -1 that fp32 GELU has, like torch's own bf16 GELU);
  lm heads (bf16 model, f32 logits of a bf16 linear output): |got - ref| <= dev  -- bit-equal unless a midpoint is in reach;
  f32 model dtype: |got - ref| <= dev + 2^-20 (|y| + |ref|), dev = the largest change of the epilogue over y +- (E_acc + E_ln)
           (no bf16 roundings; 2^-20 as above, and the fp32 rounding of the residual sum).

Inputs are chosen to see bugs: residual-stream rows with per-row mean offsets and four features 50-100x the rest, gamma
log-uniform over [0.05, 20] and beta of order 1, an all-zero row (LayerNorm gives exactly beta: the fold must give beta W with
no rstd-amplified noise), a constant non-zero row, weight rows with outliers.  Every output buffer carries NaN rows past M that
must stay NaN.  The host tests check that each modelled kernel bug moves the reference by more than 4x the bar on some element of
its case: a case that cannot see its bug is not doing its job.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import math

import numpy as np
import pytest
import torch

from oracle.config import decoder_cfg

U = 2.0 ** -24
STORE, ACT, RESIDUAL, F32 = 0, 1, 2, 3
ACT_CODE = {"gelu": 0, "relu": 1, "silu": 2, "gelu_pytorch_tanh": 3}
DEV = "cuda"

# name: (H, heads, kv heads, cross kv heads, F, activation, vocab, codebooks)
SHAPES = {
    "mini": (1024, 16, 16, 16, 4096, "gelu", 1088, 9),
    "h768": (768, 12, 12, 12, 3072, "gelu_pytorch_tanh", 1088, 9),
    "large": (1536, 24, 24, 24, 6144, "gelu", 1088, 9),
    "gqa": (1024, 16, 4, 2, 4096, "silu", 1088, 9),
    # K = H of 1..5 wgmma K stages (64 wide): short of, at and past the 3-stage ring
    "s64": (64, 1, 1, 1, 256, "gelu_pytorch_tanh", 64, 2),
    "s128": (128, 2, 2, 2, 512, "relu", 64, 2),
    "s192": (192, 3, 3, 3, 768, "silu", 64, 2),
    "s256": (256, 4, 4, 4, 1024, "gelu", 64, 2),
    "s320": (320, 5, 5, 5, 1280, "gelu", 64, 2),
}

# (name, tensor id, state-dict keys of the fused rows, LayerNorm in front, epilogue)
_L = "decoder.model.decoder.layers.0."
MATRICES = [
    ("qkv", 4, [_L + f"self_attn.{n}_proj.weight" for n in "qkv"], _L + "self_attn_layer_norm", STORE),
    ("o", 7, [_L + "self_attn.out_proj.weight"], None, RESIDUAL),
    ("q_cross", 10, [_L + "encoder_attn.q_proj.weight"], _L + "encoder_attn_layer_norm", STORE),
    ("kv_cross", 11, [_L + f"encoder_attn.{n}_proj.weight" for n in "kv"], None, STORE),
    ("o_cross", 13, [_L + "encoder_attn.out_proj.weight"], None, RESIDUAL),
    ("fc1", 16, [_L + "fc1.weight"], _L + "final_layer_norm", ACT),
    ("fc2", 17, [_L + "fc2.weight"], None, RESIDUAL),
    ("lm_heads", 20, None, "decoder.model.decoder.layer_norm", F32),
]
DECODE_M = [1, 2, 31, 32, 33, 64, 65]
PREFILL_M = [128, 129, 255, 256, 257, 1056, 2048]
CONTINUATION_M = 32 * (32 + 2050)
WORST: dict = {}       # (kernel, dtype) -> worst |got - ref| / bar over the module


def shape_cfg(name):
    H, nh, nkv, nckv, F, act, V, K = SHAPES[name]
    return decoder_cfg(hidden_size=H, num_attention_heads=nh, num_key_value_heads=nkv, num_cross_attention_key_value_heads=nckv,
                       ffn_dim=F, activation_function=act, vocab_size=V, num_codebooks=K, num_hidden_layers=1,
                       max_position_embeddings=16)


# ---- weights and inputs ------------------------------------------------------------------------------------------------
def make_weights(cfg, seed: int) -> dict:
    """fp32 state dict of a one-layer decoder: weight rows with outliers, gamma log-uniform over [0.05, 20], beta ~ N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    H, F, V, K = cfg.hidden_size, cfg.ffn_dim, cfg.vocab_size, cfg.num_codebooks
    kvH, ckvH = cfg.num_key_value_heads * 64, cfg.num_cross_attention_key_value_heads * 64

    def mat(n, k):
        w = torch.randn(n, k, generator=g) * 0.02
        rows = torch.arange(5, n, 13)
        w[rows, (rows * 7) % k] *= 40.0
        return w

    def ln(name):
        w[name + ".weight"] = torch.exp(torch.empty(H).uniform_(math.log(0.05), math.log(20.0), generator=g))
        w[name + ".bias"] = torch.randn(H, generator=g)

    p = "decoder.model.decoder."
    w = {f"{p}embed_tokens.{k}.weight": torch.zeros(V + 1, H) for k in range(K)}
    for n, (r, c) in {"self_attn.q_proj": (H, H), "self_attn.k_proj": (kvH, H), "self_attn.v_proj": (kvH, H),
                      "self_attn.out_proj": (H, H), "encoder_attn.q_proj": (H, H), "encoder_attn.k_proj": (ckvH, H),
                      "encoder_attn.v_proj": (ckvH, H), "encoder_attn.out_proj": (H, H), "fc1": (F, H), "fc2": (H, F)}.items():
        w[_L + n + ".weight"] = mat(r, c)
    for n in ("self_attn_layer_norm", "encoder_attn_layer_norm", "final_layer_norm"):
        ln(_L + n)
    ln(p + "layer_norm")
    for k in range(K):
        w[f"decoder.lm_heads.{k}.weight"] = mat(V, H)
    return w


def matrix_of(w: dict, cfg, keys) -> torch.Tensor:
    if keys is None:
        return torch.cat([w[f"decoder.lm_heads.{k}.weight"] for k in range(cfg.num_codebooks)])
    return torch.cat([w[k] for k in keys])


def residual_rows(g, M: int, K: int, offset_sigma: float | None = None) -> torch.Tensor:
    """Residual-stream rows: per-row mean offset and scale, four features 50-100x the rest; row 3 all zero, row 5 constant.
    offset_sigma: every row's mean is offset_sigma x its standard deviation instead (the LayerNorm offset sweep)."""
    scale = torch.exp(torch.randn(M, 1, generator=g) * 0.5)
    x = torch.randn(M, K, generator=g) * scale
    if offset_sigma is not None:
        x = x - x.mean(1, keepdim=True)
        x = x / x.std(1, keepdim=True) * scale
        sign = torch.where(torch.rand(M, 1, generator=g) < 0.5, -1.0, 1.0)
        return x + sign * offset_sigma * scale
    x = x + torch.randn(M, 1, generator=g) * 2.0 * scale
    feats = torch.tensor([1, K // 3, K // 2 + 1, K - 2])
    x[:, feats] *= torch.empty(len(feats)).uniform_(50.0, 100.0, generator=g)
    if M > 5:
        x[3] = 0.0
        x[5] = 1.5
    return x


def other_rows(g, M: int, K: int) -> torch.Tensor:
    """Inputs of the matrices without LayerNorm (attention output, fc1 activations): N(0, 1) rows, a few 30x features."""
    x = torch.randn(M, K, generator=g)
    x[:, torch.arange(7, K, max(1, K // 5))] *= 30.0
    return x


# ---- the reference ------------------------------------------------------------------------------------------------------
def bf16(t: torch.Tensor) -> torch.Tensor:
    return t.float().bfloat16().double()


def act_f64(v: torch.Tensor, code: int) -> torch.Tensor:
    if code == 0:
        return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))
    if code == 1:
        return v.clamp(min=0.0)
    if code == 2:
        return v * torch.sigmoid(v)
    return 0.5 * v * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (v + 0.044715 * v ** 3)))


@dataclasses.dataclass
class Layer:
    """One matrix of a case as the kernel sees it (float64 holding model-dtype values)."""
    W: torch.Tensor                 # [N, K] the packed weights (bf16 of the state dict for bf16)
    gamma: torch.Tensor | None      # [K] fp32 values, None without LayerNorm
    beta: torch.Tensor | None
    epi: int
    act: int
    bf16: bool
    eps: float = 1e-5

    @property
    def Wf(self):                   # the folded weights ptts_decoder_finalize leaves in the blob
        return (self.gamma.float() * self.W.float()).bfloat16().double()


def linear_f64(layer: Layer, x: torch.Tensor, bug: str | None = None, folded: bool = False):
    """Exact pre-epilogue output y [M, N] and the bound E on the kernel's fp32 deviation from it.  folded (bf16 with
    LayerNorm): y is the folded layer r sum_k (x_k - mu) W'_k + c2 itself, exact, and E has no E_fold term."""
    W, K = layer.W, layer.W.shape[1]
    if layer.gamma is None:
        xh = x
        y = x @ W.T
        mass = x.abs() @ W.abs().T
        e_fold = e_ln = 0.0
    else:
        mu = x.mean(1, keepdim=True)
        var = ((x - mu) ** 2).mean(1, keepdim=True)
        if bug == "unbiased_var":
            var = var * K / (K - 1)
        r = 1.0 / torch.sqrt(var + layer.eps)
        g = {"gamma_twice": layer.gamma ** 2, "no_gamma": torch.ones_like(layer.gamma)}.get(bug, layer.gamma)
        xh = (x - mu) * r * g + layer.beta
        y = xh @ W.T
        c1 = (layer.gamma[None, :] * W).sum(1)[None, :]
        c2 = (layer.beta @ W.T)[None, :]
        if bug == "no_mu_c1":
            y = y + r * mu * c1
        if bug == "no_c2":
            y = y - c2
        if layer.bf16:
            Wf = layer.Wf
            mass = r * (x.abs() @ Wf.abs().T + mu.abs() * Wf.abs().sum(1)[None, :]) + layer.beta.abs() @ W.abs().T
            shift = r * ((x - mu) @ (Wf - layer.gamma[None, :] * W).T)
            e_fold = shift.abs()
            if folded:
                y, e_fold = y + shift, 0.0
        else:
            mass = xh.abs() @ W.abs().T
            e_fold = 0.0
        e_ln = 4 * U * (K / 32 + 16) * ((y - c2).abs() + r * x.abs().mean(1, keepdim=True) * c1.abs())
    if bug in ("drop_k_first", "drop_k_last"):
        s = slice(0, 64) if bug == "drop_k_first" else slice(K - 64, K)
        y = y - xh[:, s] @ W[:, s].T
    n = K / 16 + 32 if layer.bf16 else K + 64
    return y, U * n * mass + e_fold + e_ln


def reference(layer: Layer, x: torch.Tensor, res: torch.Tensor | None, bug: str | None = None, tile: int = 128):
    """(ref, bar) [M, N]: the layer in float64 and the per-element bar of the module docstring.  bug: a modelled kernel bug
    (host sensitivity tests); the bar is always the correct layer's."""
    if bug == "tail_rows":    # the rows of the last (partial) row tile read the row above
        t0 = ((x.shape[0] - 1) // tile) * tile
        x = x.clone()
        x[t0:] = x[t0 - 1:-1].clone()
        bug = None
    y, E = linear_f64(layer, x, bug if bug in ("unbiased_var", "gamma_twice", "no_gamma", "no_mu_c1", "no_c2",
                                               "drop_k_first", "drop_k_last") else None)
    code = 3 if bug == "tanh_gelu" else layer.act
    r = None if bug == "no_residual" else res

    def epi(v):
        if layer.epi == ACT:
            return act_f64(v, code)
        if layer.epi == RESIDUAL:
            return v if r is None else r + v
        return v

    if not layer.bf16:
        ref = epi(y)
        dev = torch.maximum((epi(y - E) - ref).abs(), (epi(y + E) - ref).abs())
        bar = dev + 2.0 ** -20 * (y.abs() + ref.abs()) + 1e-30
    else:
        y1 = bf16(y)
        reach = E + 2 * U * y.abs()
        ref = epi(y1)
        dev = torch.maximum((epi(bf16(y - reach)) - ref).abs(), (epi(bf16(y + reach)) - ref).abs())
        if layer.epi == F32:
            bar = dev + 1e-30
        else:
            bar = dev + 2.0 ** -8 * (ref.abs() + dev) + 2.0 ** -20 * (y1.abs() + ref.abs()) + 1e-30
    if bug == "swap_cols":
        ref = ref.view(ref.shape[0], -1, 2).flip(-1).reshape(ref.shape)
    return ref, bar


# ---- cases --------------------------------------------------------------------------------------------------------------
def make_inputs(cfg, mat, M: int, dtype, seed: int, offset_sigma=None):
    """(x, res) on the host in the model dtype for matrix `mat` (an entry of MATRICES)."""
    name, tid, keys, ln, epi = mat
    g = torch.Generator().manual_seed(seed)
    K = cfg.ffn_dim if name == "fc2" else cfg.hidden_size
    x = residual_rows(g, M, K, offset_sigma) if ln is not None else other_rows(g, M, K)
    res = None
    if epi == RESIDUAL:
        res = residual_rows(g, M, cfg.hidden_size).to(dtype)
    return x.to(dtype), res


def make_layer(cfg, w, mat, dtype) -> Layer:
    name, tid, keys, ln, epi = mat
    is_bf16 = dtype == torch.bfloat16
    W = matrix_of(w, cfg, keys).to(dtype).double()
    gamma = w[ln + ".weight"].double() if ln else None
    beta = w[ln + ".bias"].double() if ln else None
    return Layer(W, gamma, beta, epi, ACT_CODE[cfg.activation_function], is_bf16)


# ---- host-only sensitivity tests ----------------------------------------------------------------------------------------
SENSITIVITY = [   # (bug, shape, matrix, M, row tile)
    ("drop_k_first", "s320", "qkv", 257, 128),
    ("drop_k_last", "s320", "qkv", 257, 128),
    ("drop_k_first", "mini", "fc2", 33, 32),
    ("drop_k_last", "mini", "fc2", 33, 32),
    ("tail_rows", "s256", "qkv", 257, 128),
    ("tail_rows", "s256", "o", 65, 32),
    ("no_mu_c1", "s256", "qkv", 257, 128),
    ("no_c2", "s256", "q_cross", 257, 128),
    ("gamma_twice", "s256", "fc1", 257, 128),
    ("no_gamma", "s256", "fc1", 257, 128),
    ("unbiased_var", "s64", "qkv", 257, 128),
    ("no_residual", "s256", "fc2", 257, 128),
    ("no_residual", "s256", "o_cross", 65, 32),
    ("tanh_gelu", "s256", "fc1", 257, 128),
    ("tanh_gelu", "mini", "fc1", 65, 32),
    ("swap_cols", "s256", "o", 257, 128),
    ("swap_cols", "mini", "lm_heads", 65, 32),
]
SENSITIVITY_F32 = [   # the f32 model dtype's bar (linear_f32_kernel: 32-row tiles)
    ("drop_k_first", "mini", "qkv", 65, 32),
    ("drop_k_last", "mini", "fc2", 33, 32),
    ("tail_rows", "mini", "qkv", 65, 32),
    ("gamma_twice", "mini", "fc1", 65, 32),
    ("no_gamma", "mini", "q_cross", 65, 32),
    ("unbiased_var", "s64", "qkv", 65, 32),
    ("no_residual", "mini", "o", 65, 32),
    ("tanh_gelu", "mini", "fc1", 65, 32),
    ("swap_cols", "mini", "lm_heads", 65, 32),
]


@pytest.mark.parametrize("bug,shape,mname,M,tile,dtype", [c + (torch.bfloat16,) for c in SENSITIVITY] +
                         [c + (torch.float32,) for c in SENSITIVITY_F32])
def test_reference_sees_bug(bug, shape, mname, M, tile, dtype):
    cfg = shape_cfg(shape)
    w = make_weights(cfg, seed=11)
    mat = next(m for m in MATRICES if m[0] == mname)
    layer = make_layer(cfg, w, mat, dtype)
    x, res = make_inputs(cfg, mat, M, dtype, seed=3)
    x = x.double()
    res = None if res is None else res.double()
    ref, bar = reference(layer, x, res, tile=tile)
    bad, _ = reference(layer, x, res, bug=bug, tile=tile)
    ratio = float(((bad - ref).abs() / bar).max())
    assert ratio > 4.0, f"{bug} on {shape}/{mname} moves the reference by only {ratio:.2f}x the bar"


def test_decode_shapes_reach_every_ntile_variant():
    """The decode shapes below select all six n-tile instantiations of launch_linear on a 132-SM H100 (the GPU test repeats
    this with the device's SM count)."""
    assert ntile_variants(132) == {1, 2, 3, 4, 6, 8}


def ntile_pick(N: int, sm_count: int) -> int:
    """launch_linear's rule (gemm.cu): the largest n-tile count that still gives ~one CTA per SM."""
    ntiles = N // 8
    want = min(ntiles, sm_count * 85 // 100)
    for c in (8, 6, 4, 3, 2, 1):
        if ntiles % c == 0 and ntiles // c >= want:
            return c
    return 1


def n_of(cfg, mname: str) -> int:
    """Rows of the fused matrix the hook computes for MATRICES entry `mname`."""
    H, F = cfg.hidden_size, cfg.ffn_dim
    return {"qkv": (cfg.num_attention_heads + 2 * cfg.num_key_value_heads) * 64, "o": H, "q_cross": H,
            "kv_cross": 2 * cfg.num_cross_attention_key_value_heads * 64, "o_cross": H, "fc1": F, "fc2": H,
            "lm_heads": cfg.vocab_size * cfg.num_codebooks}[mname]


def ntile_variants(sm_count):
    return {ntile_pick(n_of(shape_cfg(s), m[0]), sm_count) for s in ("mini", "h768", "large", "gqa") for m in MATRICES}


# ---- GPU -------------------------------------------------------------------------------------------------------------------
_ENGINES: dict = {}


def engine(shape, dtype, cfg=None, weights=None):
    """(cfg, weights, DecoderEngine) of SHAPES entry `shape`, or of `cfg` (a decoder config) under the name `shape`, with
    weights(cfg) instead of make_weights(cfg, seed=11) when given."""
    from parler_tts_b200.modeling import DecoderEngine
    from tests.helpers import product_decoder_config
    key = (shape, dtype)
    if key not in _ENGINES:
        _ENGINES.clear()
        cfg = shape_cfg(shape) if cfg is None else cfg
        w = make_weights(cfg, seed=11) if weights is None else weights(cfg)
        _ENGINES[key] = (cfg, w, DecoderEngine(product_decoder_config(cfg), DEV, dtype).load_state_dict(w))
    return _ENGINES[key]


def run_hook(eng, mat, x, res, M: int, path: int, pad: int, in_place: bool = False, stats_out: list | None = None):
    """The hook over the first M rows of x; the output buffer has `pad` NaN rows past M.  Returns the device output [M+pad, N]
    (and appends path 1's (mean, rstd) row statistics [M, 2] to stats_out when given)."""
    from parler_tts_b200 import _lib
    name, tid, keys, ln, epi = mat
    N = n_of(eng.cfg, name)
    dt = torch.float32 if (epi == F32 or eng.dtype == torch.float32) else torch.bfloat16
    y = torch.full((M + pad, N), float("nan"), dtype=dt, device=DEV)
    xd = x[:M].to(DEV).contiguous()
    rd = None
    if res is not None:
        if in_place:
            y[:M] = res[:M].to(DEV)
            rd = y
        else:
            rd = res[:M].to(DEV).contiguous()
    stats = torch.empty(2 * M, dtype=torch.float32, device=DEV) if (path == 1 and ln) else None
    _lib.check(_lib.lib().ptts_op_linear2(C.byref(eng.c), _lib.ptr(eng.blob), tid, 0, _lib.ptr(xd), M, 1 if ln else 0, epi,
                                          _lib.ptr(rd), _lib.ptr(y), path, _lib.ptr(stats), _lib.stream_ptr()))
    torch.cuda.synchronize()
    if stats_out is not None and stats is not None:
        stats_out.append(stats.view(M, 2).double().cpu())
    return y


def check(tag, got, ref, bar, what):
    """got [R, N] (host float64) against the reference; records the worst ratio under tag."""
    ratio = (got - ref).abs() / bar
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, float("inf")), ratio)
    worst = float(ratio.max())
    WORST[tag] = max(WORST.get(tag, 0.0), worst)
    if worst > 1.0:
        i = int(ratio.flatten().argmax())
        r, c = divmod(i, ratio.shape[1])
        raise AssertionError(f"{what}: |got - ref| = {worst:.2f} x bar at row {r} col {c}: got {float(got[r, c])!r} "
                             f"ref {float(ref[r, c])!r} bar {float(bar[r, c]):.3e} ({int((ratio > 1).sum())} elements over)")


def check_sentinels(y, M, what):
    assert torch.isnan(y[M:].float()).all(), f"{what}: rows past M = {M} were written"


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if WORST:
        print("\n[linear reference] worst |got - ref| / bar: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(WORST.items())))


@pytest.mark.gpu
def test_decode_ntile_coverage_on_this_device():
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    assert ntile_variants(sm) == {1, 2, 3, 4, 6, 8}, f"the decode shapes miss n-tile variants at {sm} SMs"


@pytest.mark.gpu
@pytest.mark.parametrize("shape,dtype", [("mini", torch.bfloat16), ("h768", torch.bfloat16), ("large", torch.bfloat16),
                                         ("gqa", torch.bfloat16), ("mini", torch.float32)])
def test_decode_gemm(shape, dtype):
    """Path 0 (launch_linear): every matrix including the lm heads, M in DECODE_M (32-row tiles: 1 row, full, one past)."""
    cfg, w, eng = engine(shape, dtype)
    tag = "decode_gemm " + ("bf16" if dtype == torch.bfloat16 else "f32")
    Mmax = max(DECODE_M)
    for j, mat in enumerate(MATRICES):
        layer = make_layer(cfg, w, mat, dtype)
        x, res = make_inputs(cfg, mat, Mmax, dtype, seed=100 + j)
        ref, bar = reference(layer, x.double(), None if res is None else res.double())
        for M in DECODE_M:
            y = run_hook(eng, mat, x, res, M, path=0, pad=32)
            what = f"{shape} {dtype} {mat[0]} M={M}"
            check_sentinels(y, M, what)
            check(tag, y[:M].double().cpu(), ref[:M], bar[:M], what)


def _prefill_rows(Ms, Mmax, seed):
    """Rows the wgmma tests compare for the Mini shape: the first tile, the last tile of every M, 64 random rows."""
    rows = set(range(128))
    for M in Ms:
        rows.update(range(((M - 1) // 128) * 128, M))
    g = torch.Generator().manual_seed(seed)
    rows.update(torch.randint(0, Mmax, (64,), generator=g).tolist())
    return torch.tensor(sorted(rows))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["s64", "s128", "s192", "s256", "s320", "mini"])
def test_wgmma_gemm(shape):
    """Path 1 (launch_linear_tc): M in PREFILL_M, every layer matrix; residual both into a separate buffer and in place."""
    cfg, w, eng = engine(shape, torch.bfloat16)
    Mmax = max(PREFILL_M)
    for j, mat in enumerate(MATRICES[:-1]):
        layer = make_layer(cfg, w, mat, torch.bfloat16)
        x, res = make_inputs(cfg, mat, Mmax, torch.bfloat16, seed=200 + j)
        rows = torch.arange(Mmax) if shape != "mini" else _prefill_rows(PREFILL_M, Mmax, seed=j)
        ref, bar = reference(layer, x[rows].double(), None if res is None else res[rows].double())
        for M in PREFILL_M:
            for in_place in ([False, True] if mat[4] == RESIDUAL else [False]):
                y = run_hook(eng, mat, x, res, M, path=1, pad=128, in_place=in_place)
                what = f"{shape} {mat[0]} M={M}{' in place' if in_place else ''}"
                check_sentinels(y, M, what)
                sel = rows < M
                check("wgmma_gemm bf16", y[rows[sel].to(DEV)].double().cpu(), ref[sel], bar[sel], what)


@pytest.mark.gpu
@pytest.mark.parametrize("mname", ["qkv", "fc2"])
def test_wgmma_gemm_continuation_size(mname):
    """A continuation prefill's M = 32 (32 + 2050) on the Mini shape: every row of the first and last tiles, 256 random rows."""
    cfg, w, eng = engine("mini", torch.bfloat16)
    mat = next(m for m in MATRICES if m[0] == mname)
    M = CONTINUATION_M
    layer = make_layer(cfg, w, mat, torch.bfloat16)
    x, res = make_inputs(cfg, mat, M, torch.bfloat16, seed=300)
    g = torch.Generator().manual_seed(301)
    rows = torch.tensor(sorted(set(range(128)) | set(range(((M - 1) // 128) * 128, M)) |
                               set(torch.randint(0, M, (256,), generator=g).tolist())))
    ref, bar = reference(layer, x[rows].double(), None if res is None else res[rows].double())
    y = run_hook(eng, mat, x, res, M, path=1, pad=128, in_place=res is not None)
    check_sentinels(y, M, f"mini {mname} M={M}")
    check("wgmma_gemm bf16", y[rows.to(DEV)].double().cpu(), ref, bar, f"mini {mname} M={M}")


@pytest.mark.gpu
def test_wgmma_hook_refuses_what_the_prefill_would_not_take():
    from parler_tts_b200 import _lib
    cfg, w, eng = engine("s128", torch.bfloat16)
    qkv, head = MATRICES[0], MATRICES[-1]
    x, _ = make_inputs(cfg, qkv, 256, torch.bfloat16, seed=1)
    with pytest.raises(ValueError):                       # M < 128
        run_hook(eng, qkv, x, None, 127, path=1, pad=0)
    with pytest.raises(ValueError):                       # the lm heads: f32 epilogue
        run_hook(eng, head, x, None, 128, path=1, pad=0)
    with pytest.raises(ValueError, match="row-major"):    # the lm heads with a bf16 epilogue: no row-major copy
        run_hook(eng, (head[0], head[1], head[2], head[3], STORE), x, None, 128, path=1, pad=0)
    cfg32, w32, eng32 = engine("s128", torch.float32)
    with pytest.raises(ValueError):                       # f32 model dtype
        run_hook(eng32, qkv, x.float(), None, 128, path=1, pad=0)
    with pytest.raises(ValueError):
        _lib.check(_lib.lib().ptts_op_linear2(C.byref(eng32.c), _lib.ptr(eng32.blob), 4, 0, _lib.ptr(x[:128].float().to(DEV)),
                                              128, 1, 0, None, _lib.ptr(torch.empty(128, 384, device=DEV)), 2, None,
                                              _lib.stream_ptr()))


@pytest.mark.gpu
def test_original_signature_is_the_decode_gemm():
    """ptts_op_linear (the signature before `path` existed) is ptts_op_linear2 with path 0: bit-identical outputs."""
    from parler_tts_b200 import _lib
    cfg, w, eng = engine("s256", torch.bfloat16)
    for j, mat in enumerate(MATRICES):
        x, res = make_inputs(cfg, mat, 45, torch.bfloat16, seed=500 + j)
        want = run_hook(eng, mat, x, res, 45, path=0, pad=0)
        got = torch.empty_like(want)
        rd = None if res is None else res.to(DEV).contiguous()
        _lib.check(_lib.lib().ptts_op_linear(C.byref(eng.c), _lib.ptr(eng.blob), mat[1], 0, _lib.ptr(x.to(DEV).contiguous()), 45,
                                             1 if mat[3] else 0, mat[4], _lib.ptr(rd), _lib.ptr(got), _lib.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(got.view(torch.int16 if got.dtype == torch.bfloat16 else torch.int32),
                           want.view(torch.int16 if want.dtype == torch.bfloat16 else torch.int32)), mat[0]


# ---- LayerNorm statistics at large mean offsets -------------------------------------------------------------------------
LN_ASSERTED = [1.0, 4.0, 16.0]
LN_RECORDED = [32.0, 64.0, 128.0]


@pytest.mark.gpu
@pytest.mark.parametrize("path", [0, 1])
def test_layernorm_at_large_offsets(path, record_property):
    """Rows whose mean is |mu|/sigma = 1 .. 16 standard deviations away from 0 pass the bar on both paths (the decode path
    computes var = S2/K - mu^2 in one pass); 32, 64 and 128 are measured and recorded, not asserted.

    The bar grows with |mu|/sigma through the fold's cancellation term, so the error-to-bar ratio alone does not measure the
    statistics.  Two more numbers are recorded per offset: the rstd the kernel effectively applied, relative to the exact one
    (per row, the least-squares scale of got - c2 against the exact r sum_k (x_k - mu) W'_k over the 3072 outputs, which
    averages the outputs' bf16 rounding down), and for path 1 the rstd row_stats_kernel wrote, which gives the fit's own noise
    floor by comparison.  ln_stats.cuh estimates var's relative error of the one-pass
    form as ~1e-6 (1 + mu^2 / sigma^2), i.e. ~5e-7 (1 + mu^2 / sigma^2) on rstd."""
    cfg, w, eng = engine("mini", torch.bfloat16)
    mat = MATRICES[0]
    layer = make_layer(cfg, w, mat, torch.bfloat16)
    M, pad = (64, 32) if path == 0 else (256, 128)
    worst, fit, direct = {}, {}, {}
    for k, off in enumerate(LN_ASSERTED + LN_RECORDED):
        x, _ = make_inputs(cfg, mat, M, torch.bfloat16, seed=400 + k, offset_sigma=off)
        xd = x.double()
        ref, bar = reference(layer, xd, None)
        stats = []
        y = run_hook(eng, mat, x, None, M, path=path, pad=pad, stats_out=stats)
        check_sentinels(y, M, f"offset {off} path {path}")
        got = y[:M].double().cpu()
        ratio = float(((got - ref).abs() / bar).max())
        assert math.isfinite(ratio), f"path {path}, |mu|/sigma = {off}: non-finite output"
        worst[off] = ratio
        # the effective rstd: the kernel computes r (sum_k x_k W'_k - mu c1) + c2 = r sum_k (x_k - mu) W'_k + c2, so got - c2
        # scales with the kernel's r against the exact r sum_k (x_k - mu) W'_k (with the folded W', so that the fold's rounding
        # does not enter the fit)
        mu = xd.mean(1, keepdim=True)
        r = 1.0 / torch.sqrt(((xd - mu) ** 2).mean(1, keepdim=True) + layer.eps)
        z = r * ((xd - mu) @ layer.Wf.T)
        c2 = (layer.beta @ layer.W.T)[None, :]
        rho = ((got - c2) * z).sum(1) / (z ** 2).sum(1)
        fit[off] = float((rho - 1).abs().max())
        record_property(f"path{path}_offset{int(off)}_worst_ratio", ratio)
        record_property(f"path{path}_offset{int(off)}_fitted_rstd_rel_err", fit[off])
        if stats:
            direct[off] = float((stats[0][:, 1:] / r - 1).abs().max())
            record_property(f"path{path}_offset{int(off)}_rstd_rel_err", direct[off])
    print(f"\n[linear reference] LayerNorm offset sweep, path {path} (|mu|/sigma: error/bar, fitted rstd error"
          f"{', row_stats rstd error' if direct else ''}): " +
          "; ".join(f"{int(o)}: {worst[o]:.3f}, {fit[o]:.2e}" + (f", {direct[o]:.2e}" if direct else "") for o in worst))
    for off in LN_ASSERTED:
        assert worst[off] <= 1.0, f"path {path}: |mu|/sigma = {off} exceeds the bar ({worst[off]:.2f}x)"
