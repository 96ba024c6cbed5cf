"""References of the text encoders' own kernels (csrc/text.cu: rownorm, ewise, embed, gather_rows and the T5 gated
half), their named mutations, the fixtures the operator tests run, and the ctypes binding of the test hooks that launch
them (csrc/rf_api.cu: rf_dbg_text_*, rf_dbg_t5_gated_gelu).

Values are fp32 tensors holding bf16 values.  Each reference is the transformers module's arithmetic restated in fp32
(float64 for LayerNorm's statistics) with a bf16 rounding wherever eager bf16 torch rounds:

  * T5LayerNorm: bf16(w * bf16(x * rsqrt(mean(x^2) + eps))), statistics in fp32;
  * affine LayerNorm (CLIP, eps 1e-5): one rounding of (x - mean) / sqrt(var + eps) * w + b;
  * NewGELUActivation ("gelu_new", T5-v1.1's dense_act_fn): every op of
    0.5 * x * (1 + tanh(sqrt(2/pi) * (x + 0.044715 * pow(x, 3)))) rounds, pow(x, 3) as bf16(bf16(x x) x); the
    T5 feed-forward multiplies the result by bf16(x wi_1^T) and rounds once more;
  * QuickGELUActivation (CLIP): bf16(x * bf16(sigmoid(bf16(1.702 x))));
  * embeddings: a row gather, + the position row t % S with one bf16 add (CLIPTextEmbeddings); the pooled rows of CLIP
    are the rows b S + pos[b].

`mut` names one deliberate change from MUTATIONS; the host tests show each one moves a fixture the GPU tests run."""
import ctypes
from ctypes import c_float, c_int, c_int64, c_void_p

import torch

from tests import _exact as E
from tests._exact import bf, f32

BF = torch.bfloat16
T5_EPS = 1e-6   # T5-v1.1's layer_norm_epsilon, what rf_t5_encode passes
CLIP_EPS = 1e-5  # CLIP's layer_norm_eps, what rf_clip_encode passes
GELU_C = f32(0.044715)
GELU_S = f32(0.7978845608028654)  # sqrt(2 / pi) as torch takes a Python float into an fp32 multiply
QUICK_C = f32(1.702)

MUTATIONS = {
    "gelu_fused": "the DiT's fused GELU-tanh (one rounding) instead of gelu_new's eager chain",
    "cube_once": "pow(x, 3) rounded once instead of bf16(bf16(x x) x)",
    "rms_unrounded": "T5LayerNorm without the bf16 rounding of the normalised value before * w",
    "ln_eps": "LayerNorm eps 1e-6 instead of 1e-5",
    "ln_no_mean": "LayerNorm without the mean subtraction",
    "quick_unrounded": "quick-GELU without its inner bf16 roundings",
    "pos_row_t": "position row t instead of t % S",
    "gather_batch0": "pooled rows gathered from batch 0's rows",
}


# ------------------------------------------------------------------------------------ row norms
def t5_layernorm(x, w, eps=T5_EPS, mut=()):
    xf = x.float()
    var = xf.pow(2).mean(-1, keepdim=True)
    h = xf * torch.rsqrt(var + eps)
    if "rms_unrounded" not in mut:
        h = bf(h)
    return bf(w.float() * h)


def layer_norm(x, w, b, eps=CLIP_EPS, mut=()):
    xd = x.double()
    mean = torch.zeros_like(xd[..., :1]) if "ln_no_mean" in mut else xd.mean(-1, keepdim=True)
    var = (xd - mean).pow(2).mean(-1, keepdim=True)
    y = (xd - mean) / torch.sqrt(var + (1e-6 if "ln_eps" in mut else eps)) * w.double() + b.double()
    return bf(y.float())


# ------------------------------------------------------------------------------------ activations
def gelu_new(a, mut=()):
    x = a.float()
    if "gelu_fused" in mut:
        return E.gelu(x)
    p = bf(x * x * x) if "cube_once" in mut else bf(bf(x * x) * x)
    q = bf(GELU_C.to(x.device) * p)
    r = bf(x + q)
    s = bf(GELU_S.to(x.device) * r)
    t = bf(torch.tanh(s))
    u = bf(1.0 + t)
    h = bf(0.5 * x)
    return bf(h * u)


def gated(a, b, mut=()):
    """T5DenseGatedActDense's hidden_gelu * hidden_linear"""
    return bf(gelu_new(a, mut) * b.float())


def quick_gelu(a, mut=()):
    x = a.float()
    c = QUICK_C.to(x.device)
    if "quick_unrounded" in mut:
        return bf(x * torch.sigmoid(c * x))
    return bf(x * bf(torch.sigmoid(bf(c * x))))


# ------------------------------------------------------------------------------------ gathers
def embed(ids, table, pos=None, S=None, mut=()):
    """ids [T] -> table rows [T, D] (+ pos[t % S] with one bf16 add)"""
    rows = table[ids.long()].float()
    if pos is None:
        return rows
    t = torch.arange(ids.numel(), device=ids.device)
    idx = t % pos.shape[0] if "pos_row_t" in mut else t % S
    return bf(rows + pos[idx].float())


def gather(x, pos, S, mut=()):
    """x [B S, D], pos [B] -> x[b S + pos[b]]"""
    b = torch.arange(pos.numel(), device=pos.device)
    return x[pos.long() if "gather_batch0" in mut else b * S + pos.long()].float()


# ------------------------------------------------------------------------------------ fixtures
NORM_DIMS = (256, 768, 1024, 4096)
NORM_ROWS = (1, 7, 77, 231, 1031)  # not multiples of the 8 rows a block covers
# unit rows; |x| ~ 1e3 (T5's late-layer residual); std 2^-6 (eps a visible part of the variance); one all-zero row;
# one dominant element per row; mean / std = 128 (LayerNorm only)
NORM_CASES = {0: ("unit", "large", "small", "zero_row", "dominant"),
              1: ("unit", "large", "small", "zero_row", "dominant", "offset")}


def norm_inputs(rows, dim, case, mode):
    """(x [rows, dim], w [dim], b [dim] or None) bf16 on the CPU"""
    g = torch.Generator().manual_seed(rows * 10007 + dim * 13 + mode * 7 + NORM_CASES[1].index(case))
    x = torch.randn(rows, dim, generator=g)
    if case == "large":
        x = x * 1e3
    elif case == "small":
        x = x * 2.0 ** -6
    elif case == "zero_row":
        x[rows // 2] = 0
    elif case == "dominant":
        x = x * 0.01
        j = torch.randint(0, dim, (rows,), generator=g)
        x[torch.arange(rows), j] = 300 * torch.sign(torch.randn(rows, generator=g))
    elif case == "offset":
        x = x + 128
    w = (1 + 0.1 * torch.randn(dim, generator=g)).to(BF)
    b = (0.05 * torch.randn(dim, generator=g)).to(BF) if mode == 1 else None
    return x.to(BF), w, b


def all_finite_bf16():
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(BF)
    return bits[torch.isfinite(bits.float())]


def random_pairs(n=1 << 20, seed=3):
    """(a, b): a spread over gelu_new's curved range [-8, 8] and beyond, b ~ N(0, 1)"""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(n, generator=g) * 3
    b = torch.randn(n, generator=g)
    return a.to(BF), b.to(BF)


# ------------------------------------------------------------------------------------ test-hook binding
HOOKS = {  # name -> argument types (vp: pointer, ci: int, cl: int64_t, cf: float)
    "rf_dbg_text_embed": "vp vp vp vp ci ci ci vp",
    "rf_dbg_text_rownorm": "vp vp ci ci vp vp cf ci vp",
    "rf_dbg_text_ewise": "vp vp vp cl ci vp",
    "rf_dbg_text_gather_rows": "vp vp vp ci ci ci vp",
    "rf_dbg_t5_gated_gelu": "vp ci ci vp vp ci vp vp vp",
}
_TYPES = {"vp": c_void_p, "ci": c_int, "cl": c_int64, "cf": c_float}


def declare(lib):
    for name, args in HOOKS.items():
        fn = getattr(lib, name)
        fn.restype = c_int
        fn.argtypes = [_TYPES[a] for a in args.split()]
    return lib


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())
