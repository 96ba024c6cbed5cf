"""Exact-operand references of the grouped GEMM's epilogues and of the LoRA helper kernels, plus the ctypes binding of
the test hooks that launch them (csrc/rf_api.cu: rf_dbg_*).

Operands are drawn from small dyadic grids: activations k/8 (|k| <= 8), weights and LoRA A factors k/32 (|k| <= 8),
LoRA B factors k/16 (|k| <= 4).  Every product is then a multiple of 2^-e and, as `gemm` checks, the sum of the
products' magnitudes stays below 2^(23 - e): every partial sum is exact in fp32 whatever the order and the
tensor-core alignment, so the kernel's fp32 accumulator is known exactly.  The accumulated values still need more
than 8 significant bits, so each bf16 rounding point changes bits and its position matters.

References: the GEMM in float64 (its cast to fp32 asserted exact), then the epilogue in fp32 in the kernel's order,
rounded to bf16 at the reference's rounding points (DESIGN.md section 5).  Values are fp32 tensors holding bf16
values.  With `exact=False` the same functions are high-precision references for random operands.  `mut` names one
deliberate change (see MUTATIONS) that the host tests use to show the bit-exact GPU tests would notice it."""
import ctypes
from ctypes import c_float, c_int, c_int64, c_void_p

import torch

EPI_BIAS, EPI_GELU, EPI_GATE_RES, EPI_QKV, EPI_SCALE = 0, 1, 2, 3, 4

MUTATIONS = {
    "L_unrounded": "bf16(L * s) instead of bf16(bf16(L) * s)",
    "scale_sec0": "section 0's scale used for every column section",
    "T_unrounded": "T = x A^T not rounded to bf16 before the up-projection",
    "lora_before_bias": "LoRA term added before the bias rounding",
    "merge_thrice": "merge rounded three times: bf16(W + bf16(bf16(B A) * s))",
}


def bf(x):
    """a bf16 rounding point of an fp32 value"""
    return x.to(torch.bfloat16).float()


def f32(s):
    return torch.tensor(float(s), dtype=torch.float32)


def dyadic(shape, log2_step, kmax, seed, device="cpu"):
    """bf16 tensor of k * 2^-log2_step, k uniform in [-kmax, kmax]"""
    g = torch.Generator(device=device).manual_seed(seed)
    k = torch.randint(-kmax, kmax + 1, tuple(shape), generator=g, device=device)
    return (k.double() * 2.0 ** -log2_step).to(torch.bfloat16)


def act(shape, seed, device="cpu"):
    return dyadic(shape, 3, 8, seed, device)


def weight(shape, seed, device="cpu"):
    return dyadic(shape, 5, 8, seed, device)


def lora_b(shape, seed, device="cpu"):
    return dyadic(shape, 4, 4, seed, device)


def randn(shape, seed, scale=1.0, device="cpu"):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(tuple(shape), generator=g) * scale).to(torch.bfloat16).to(device)


def lsb_exp(t):
    """least e >= 0 with every element of t a multiple of 2^-e"""
    d = t.double()
    for e in range(40):
        s = d * 2.0 ** e
        if torch.equal(s, s.round()):
            return e
    raise AssertionError("not a dyadic grid")


def gemm(a, w, exact=True):
    """a [M, K] @ w [N, K]^T in float64, returned in fp32.  exact: assert that fp32 accumulation of these operands is
    exact in any order (products on a 2^-e grid, sum of their magnitudes below 2^(23 - e)) and the cast is exact."""
    a64, w64 = a.double(), w.double()
    y = a64 @ w64.t()
    if exact:
        e = lsb_exp(a) + lsb_exp(w)
        bound = (a64.abs() @ w64.abs().t()).max().item() if y.numel() else 0.0
        assert bound < 2.0 ** (23 - e), f"operands not exact in fp32: sum |a w| = {bound} >= 2^{23 - e}"
        assert torch.equal(y.float().double(), y)
    return y.float()


def lora_down(x, A, exact=True, mut=()):
    """T = bf16(x A^T)"""
    t = gemm(x, A, exact)
    return t if "T_unrounded" in mut else bf(t)


def lora_up(T, B, scales, sec_cols, pad, exact=True, mut=()):
    """the fused term of every column section s: bf16(bf16(T[:, pad s : pad (s + 1)] B_s^T) * scales[s])"""
    N = B.shape[0]
    width = sec_cols or N
    L = torch.empty(T.shape[0], N, dtype=torch.float32, device=T.device)
    for s in range(N // width):
        cols = slice(s * width, (s + 1) * width)
        l = gemm(T[:, s * pad:(s + 1) * pad], B[cols], exact and "T_unrounded" not in mut)
        if "L_unrounded" not in mut:
            l = bf(l)
        L[:, cols] = bf(l * f32(scales[0 if "scale_sec0" in mut else s]).to(l.device))
    return L


def linear(a, w, bias=None, addend=None, L=None, exact=True, mut=()):
    """bf16(acc + bias) [-> bf16(. + addend)] [-> bf16(. + L)]"""
    y = gemm(a, w, exact)
    if bias is not None:
        y = y + bias.float()
    if L is not None and "lora_before_bias" in mut:
        y = y + L
        L = None
    y = bf(y)
    if addend is not None:
        y = bf(y + addend.float())
    if L is not None:
        y = bf(y + L)
    return y


def gate_res(v, res, gate):
    return bf(res.float() + bf(gate.float() * v))


def gelu(v):
    """GELU-tanh of the bf16 value in float64, as x sigmoid(2 u) (= 0.5 x (1 + tanh u)), rounded once to bf16.  torch's
    fp32 tanh form loses the negative tail to cancellation in 1 + tanh(u); the kernel's sigmoid form does not."""
    d = v.double()
    u = 0.7978845608028654 * (d + 0.044715 * d * d * d)
    return (d * torch.sigmoid(2.0 * u)).to(torch.bfloat16).float()


def scale_out(v, s):
    return bf(v * f32(s).to(v.device))


def qkv_post(v, cos, sin, nq, nk, heads):
    """per-head RMSNorm * w and interleaved RoPE on the q / k sections of v (fp32, bf16 values, [M, 3 heads 128]) in
    the kernel's order: lane q of a quad sums the squares of columns 8 jj + 2 q + {0, 1} of a head in jj order (v^2 is
    exact in fp32, so its fma chain is an fp32 add chain), the quad reduces as (s0 + s1) + (s2 + s3); rinv =
    1 / sqrt(ss / 128 + 1e-6) with IEEE sqrt and division; RoPE with separate fp32 multiplies and one add."""
    M = v.shape[0]
    inner = heads * 128
    out = v.clone()
    for sec, nw in ((0, nq), (1, nk)):
        t = v[:, sec * inner:(sec + 1) * inner].reshape(M, heads, 16, 4, 2)
        sq = t * t
        s = torch.zeros(M, heads, 4, dtype=torch.float32, device=v.device)
        for jj in range(16):
            for e in range(2):
                s = s + sq[:, :, jj, :, e]
        ss = (s[..., 0] + s[..., 1]) + (s[..., 2] + s[..., 3])
        var = ss / 128.0
        rinv = torch.div(torch.ones_like(var), torch.sqrt(var + 1e-6))
        y = bf(t.reshape(M, heads, 128) * rinv[..., None])
        y = bf(y * nw.float())
        y = y.view(M, heads, 64, 2)
        y0, y1 = y[..., 0], y[..., 1]
        c, sn = cos[:, None, :], sin[:, None, :]
        o0 = y0 * c + (-y1) * sn
        o1 = y1 * c + y0 * sn
        out[:, sec * inner:(sec + 1) * inner] = bf(torch.stack([o0, o1], -1).reshape(M, inner))
    return out


def add_rows(dst, src, s):
    """dst + bf16(src * s), rounded"""
    return bf(dst.float() + bf(src.float() * f32(s).to(src.device)))


def lora_merge(W, A, B, s, exact=True, mut=()):
    """bf16(W + s * (B A)), one rounding (peft's merged weight)"""
    d = gemm(B, A.t(), exact)
    sc = f32(s).to(d.device)
    if "merge_thrice" in mut:
        return bf(W.float() + bf(bf(d) * sc))
    return bf(W.float() + d * sc)


def ulps(got, ref):
    """bf16 ulps between two bf16 tensors (sign-magnitude bit patterns mapped to a monotone integer line)"""
    def line(t):
        b = t.to(torch.bfloat16).view(torch.int16).int()
        return torch.where(b < 0, -(b & 0x7FFF), b)
    return (line(got) - line(ref)).abs()


# ------------------------------------------------------------------------------------ test-hook binding
class GemmGroup(ctypes.Structure):
    """mirror of rf_dbg_gemm_group (csrc/rf_api.cu) = rf::GemmGroupArgs"""
    _fields_ = [("A", c_void_p), ("lda", c_int), ("M", c_int), ("W", c_void_p), ("bias", c_void_p),
                ("out", c_void_p), ("ldo", c_int), ("addend", c_void_p), ("ldadd", c_int),
                ("res", c_void_p), ("ldr", c_int), ("gate", c_void_p), ("rope_cos", c_void_p),
                ("rope_sin", c_void_p), ("norm_q", c_void_p), ("norm_k", c_void_p),
                ("lora_T", c_void_p), ("ld_t", c_int), ("lora_B", c_void_p), ("lora_sec_cols", c_int),
                ("lora_pad", c_int), ("lora_scale", c_float * 3)]


def declare(lib):
    vp, ci = c_void_p, c_int
    lib.rf_dbg_gemm_group_size.restype = ctypes.c_size_t
    lib.rf_dbg_gemm_group_size.argtypes = []
    lib.rf_dbg_gemm_grouped.restype = ci
    lib.rf_dbg_gemm_grouped.argtypes = [ci, ci, ci, ci, ctypes.POINTER(GemmGroup), vp]
    lib.rf_dbg_lora_down_grouped.restype = ci
    lib.rf_dbg_lora_down_grouped.argtypes = [ci, ci, ci, ctypes.POINTER(GemmGroup), vp]
    lib.rf_dbg_ln_modulate_grouped.restype = ci
    lib.rf_dbg_ln_modulate_grouped.argtypes = [vp, ci, vp, ci, ci, ci, ctypes.POINTER(ci), ctypes.POINTER(vp),
                                               ctypes.POINTER(vp), vp]
    lib.rf_dbg_add_rows.restype = ci
    lib.rf_dbg_add_rows.argtypes = [vp, c_int64, vp, ci, ci, ci, c_float, vp]
    lib.rf_dbg_lora_merge.restype = ci
    lib.rf_dbg_lora_merge.argtypes = [vp, vp, vp, vp, ci, ci, ci, c_float, vp]
    return lib


def _p(t):
    return None if t is None else t.data_ptr()


def _ld(t):
    return 0 if t is None else t.stride(0)


def group(A, W, out, bias=None, addend=None, res=None, gate=None, cos=None, sin=None, nq=None, nk=None, T=None,
          B=None, sec_cols=0, pad=0, scales=(1.0, 1.0, 1.0)):
    """one GemmGroup over torch views (row pitch = stride(0)); the caller keeps the tensors alive"""
    g = GemmGroup()
    g.A, g.lda, g.M, g.W, g.bias = _p(A), _ld(A), A.shape[0], _p(W), _p(bias)
    g.out, g.ldo = _p(out), _ld(out)
    g.addend, g.ldadd = _p(addend), _ld(addend)
    g.res, g.ldr, g.gate = _p(res), _ld(res), _p(gate)
    g.rope_cos, g.rope_sin, g.norm_q, g.norm_k = _p(cos), _p(sin), _p(nq), _p(nk)
    g.lora_T, g.ld_t, g.lora_B = _p(T), _ld(T), _p(B)
    g.lora_sec_cols, g.lora_pad = sec_cols, pad
    for i in range(3):
        g.lora_scale[i] = scales[i] if i < len(scales) else 0.0
    return g


def groups_array(groups):
    return (GemmGroup * len(groups))(*groups)
