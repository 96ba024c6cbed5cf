"""-m gpu: operator-level parity of the sm_90a kernels, called through the C ABI (ctypes), against
plain torch fp32 restatements of the same op with the reference's bf16 rounding points
(SURVEY.md Appendix A).  Tolerances are stated per test."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from reflectionflow_b200 import _lib as L  # noqa: E402


def _dev():
    return torch.device("cuda:0")


def _randn(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(_dev())


def _linear_ref(x, W, b):
    y = x.float() @ W.float().t()
    if b is not None:
        y = y + b.float()
    return y.to(torch.bfloat16)


def _report(name, got, ref, bm=128, bn=256):
    d = (got.float() - ref.float()).abs()
    print(f"[{name}] max_abs={d.max().item():.4g} mean_abs={d.mean().item():.4g} "
          f"ref_absmax={ref.float().abs().max().item():.4g}")
    if d.max().item() > 0.5 and d.dim() == 2:
        # tile map of the error, to localise descriptor / layout bugs
        M, N = d.shape
        rows = []
        for m0 in range(0, min(M, 4 * bm), 32):
            rows.append(" ".join(f"{d[m0:m0 + 32, n0:n0 + 32].max().item():7.2g}"
                                 for n0 in range(0, min(N, 256), 32)))
        print("error map (32x32 blocks, first rows/cols):\n" + "\n".join(rows))


def _call_linear(epi, x, W, bias, y, addend=None, res=None, gate=None, cos=None, sin=None,
                 nq=None, nk=None):
    lib = L.load()
    M, K = x.shape
    N = W.shape[0]
    rc = lib.rf_op_linear(epi, M, N, K, L.ptr(x), x.stride(0), L.ptr(W), L.ptr(bias), L.ptr(y),
                          y.stride(0), L.ptr(addend), addend.stride(0) if addend is not None else 0,
                          L.ptr(res), res.stride(0) if res is not None else 0, L.ptr(gate),
                          L.ptr(cos), L.ptr(sin), L.ptr(nq), L.ptr(nk), L.cur_stream())
    L.check(rc, "rf_op_linear")
    torch.cuda.synchronize()


@pytest.fixture(params=["pair", "single"])
def gemm_path(request):
    """big shapes run on 256-wide tiles; `single` forces tiles at most 128 wide so both tile widths of
    csrc/gemm_sm90.cu stay covered"""
    lib = L.load()
    lib.rf_dbg_force_gemm_v1(1 if request.param == "single" else 0)
    yield request.param
    lib.rf_dbg_force_gemm_v1(0)


@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (256, 256, 128), (200, 128, 192),
                                   (4608, 3072, 3072), (512, 3072, 4096), (4096, 64, 3072),
                                   (1024, 12288, 3072), (768, 3072, 15360), (300, 512, 256),
                                   (4608 + 77, 768, 512)])
def test_linear_bias(M, N, K, gemm_path):
    x = _randn(M, K, seed=1)
    W = _randn(N, K, scale=1.0 / math.sqrt(K), seed=2)
    b = _randn(N, seed=3)
    y = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=_dev())
    _call_linear(0, x, W, b, y)
    ref = _linear_ref(x, W, b)
    _report(f"linear {M}x{N}x{K}", y, ref)
    # fp32-accumulated bf16 GEMM: only summation order differs -> at most 1 bf16 ulp
    torch.testing.assert_close(y.float(), ref.float(), rtol=2 ** -7, atol=2e-2)
    frac_exact = (y == ref).float().mean().item()
    print(f"  bit-exact fraction {frac_exact:.4f}")
    assert frac_exact > 0.97


def test_linear_no_bias_and_addend(gemm_path):
    M, N, K = 384, 256, 256
    x = _randn(M, K, seed=4)
    W = _randn(N, K, scale=1.0 / math.sqrt(K), seed=5)
    add = _randn(M, N, seed=6)
    y = torch.empty((M, N), dtype=torch.bfloat16, device=_dev())
    _call_linear(0, x, W, None, y, addend=add)
    ref = (_linear_ref(x, W, None).float() + add.float()).to(torch.bfloat16)
    _report("linear addend", y, ref)
    torch.testing.assert_close(y.float(), ref.float(), rtol=2 ** -7, atol=2e-2)


def test_linear_gelu(gemm_path):
    M, N, K = 640, 512, 256
    x = _randn(M, K, seed=7)
    W = _randn(N, K, scale=1.0 / math.sqrt(K), seed=8)
    b = _randn(N, seed=9)
    y = torch.empty((M, N), dtype=torch.bfloat16, device=_dev())
    _call_linear(1, x, W, b, y)
    ref = torch.nn.functional.gelu(_linear_ref(x, W, b).float(), approximate="tanh").to(torch.bfloat16)
    _report("linear gelu", y, ref)
    torch.testing.assert_close(y.float(), ref.float(), rtol=2 ** -6, atol=2e-2)


def test_linear_gate_residual_inplace(gemm_path):
    M, N, K = 512, 768, 512
    x = _randn(M, K, seed=10)
    W = _randn(N, K, scale=1.0 / math.sqrt(K), seed=11)
    b = _randn(N, seed=12)
    gate = _randn(N, seed=13)
    res = _randn(M, N, seed=14)
    lin = _linear_ref(x, W, b)
    ref = (res.float() + (gate.float() * lin.float()).to(torch.bfloat16).float()).to(torch.bfloat16)
    y = res.clone()
    _call_linear(2, x, W, b, y, res=y, gate=gate)
    _report("linear gate+res", y, ref)
    torch.testing.assert_close(y.float(), ref.float(), rtol=2 ** -6, atol=3e-2)


def _rope_tables(n_tok, seed=0):
    g = torch.Generator().manual_seed(seed)
    ang = torch.rand(n_tok, 64, generator=g) * 6.28
    return ang.cos().contiguous().to(_dev()), ang.sin().contiguous().to(_dev())


def _qkv_ref(x, W, b, cos, sin, nq, nk, heads):
    return _qkv_post_ref(_linear_ref(x, W, b), cos, sin, nq, nk, heads)


def _qkv_post_ref(y, cos, sin, nq, nk, heads):
    """per-head RMSNorm * w and interleaved RoPE on the q / k sections of a bf16 [M, 3*heads*128] linear output"""
    M = y.shape[0]
    inner = heads * 128
    out = torch.empty_like(y)
    for sec, nw in ((0, nq), (1, nk)):
        t = y[:, sec * inner:(sec + 1) * inner].view(M, heads, 128)
        var = t.float().pow(2).mean(-1, keepdim=True)
        t2 = (t.float() * torch.rsqrt(var + 1e-6)).to(torch.bfloat16)
        t2 = (t2.float() * nw.float()).to(torch.bfloat16)
        xr = t2.float().view(M, heads, 64, 2)
        x0, x1 = xr[..., 0], xr[..., 1]
        c, s = cos[:, None, :], sin[:, None, :]
        o0 = x0 * c + (-x1) * s
        o1 = x1 * c + x0 * s
        out[:, sec * inner:(sec + 1) * inner] = torch.stack([o0, o1], -1).reshape(M, inner).to(torch.bfloat16)
    out[:, 2 * inner:] = y[:, 2 * inner:]
    return out


@pytest.mark.parametrize("M,heads,K", [(256, 2, 256), (640, 24, 512), (333, 4, 256)])
def test_linear_qkv_rmsnorm_rope(M, heads, K, gemm_path):
    N = 3 * heads * 128
    x = _randn(M, K, seed=20)
    W = _randn(N, K, scale=1.0 / math.sqrt(K), seed=21)
    b = _randn(N, scale=0.1, seed=22)
    nq = (1.0 + 0.1 * _randn(128, seed=23).float()).to(torch.bfloat16)
    nk = (1.0 + 0.1 * _randn(128, seed=24).float()).to(torch.bfloat16)
    cos, sin = _rope_tables(M)
    y = torch.empty((M, N), dtype=torch.bfloat16, device=_dev())
    _call_linear(3, x, W, b, y, cos=cos, sin=sin, nq=nq, nk=nk)
    ref = _qkv_ref(x, W, b, cos, sin, nq, nk, heads)
    _report("linear qkv", y, ref)
    torch.testing.assert_close(y.float(), ref.float(), rtol=2 ** -6, atol=3e-2)


def _lora_pad(A, B):
    """rank r -> zero-padded rank 64 (the C ABI's LoRA layout)"""
    r = A.shape[0]
    Ap = torch.zeros(64, A.shape[1], dtype=A.dtype, device=A.device)
    Bp = torch.zeros(B.shape[0], 64, dtype=B.dtype, device=B.device)
    Ap[:r] = A
    Bp[:, :r] = B
    return Ap.contiguous(), Bp.contiguous()


def _peft_linear_ref(x, W, b, A, B):
    """peft LoRA Linear in bf16: base -> bf16, lora_A -> bf16, lora_B -> bf16, sum -> bf16"""
    y = _linear_ref(x, W, b)
    t = (x.float() @ A.float().t()).to(torch.bfloat16)
    l = (t.float() @ B.float().t()).to(torch.bfloat16)
    return (y.float() + l.float()).to(torch.bfloat16)


def _call_linear_lora(epi, x, W, bias, y, Ap, Bp, t_cols, res=None, gate=None, cos=None, sin=None, nq=None,
                      nk=None):
    lib = L.load()
    M, K = x.shape
    N = W.shape[0]
    ws = torch.zeros(lib.rf_op_linear_lora_workspace_bytes(M), dtype=torch.uint8, device=_dev())
    rc = lib.rf_op_linear_lora(epi, M, N, K, L.ptr(x), x.stride(0), L.ptr(W), L.ptr(bias), L.ptr(y), y.stride(0),
                               L.ptr(Ap), t_cols, L.ptr(Bp), L.ptr(res), res.stride(0) if res is not None else 0,
                               L.ptr(gate), L.ptr(cos), L.ptr(sin), L.ptr(nq), L.ptr(nk), L.ptr(ws), L.cur_stream())
    L.check(rc, "rf_op_linear_lora")
    torch.cuda.synchronize()


@pytest.mark.parametrize("M,N,K", [(1024, 3072, 3072), (1024, 3072, 15360), (256, 256, 256), (1000, 1024, 12288)])
def test_linear_lora_gate_res(M, N, K):
    """fused peft-LoRA GEMM (down-projection GEMM + low-rank k-block in the main GEMM) at the
    headline condition-stream shapes: to_out / ff.net.2 / single proj_out (lora_controller.py:5-42)"""
    x = _randn(M, K, seed=70)
    W = _randn(N, K, scale=1.0 / math.sqrt(K), seed=71)
    b = _randn(N, scale=0.1, seed=72)
    A = _randn(32, K, scale=1.0 / math.sqrt(K), seed=73)
    B = _randn(N, 32, scale=0.5 / math.sqrt(32), seed=74)
    gate = _randn(N, scale=0.5, seed=75)
    res = _randn(M, N, seed=76)
    y = res.clone()
    Ap, Bp = _lora_pad(A, B)
    _call_linear_lora(2, x, W, b, y, Ap, Bp, 64, res=res.clone(), gate=gate)
    lin = _peft_linear_ref(x, W, b, A, B)
    ref = (res.float() + (gate.float()[None] * lin.float()).to(torch.bfloat16).float()).to(torch.bfloat16)
    _report("linear_lora gate_res", y, ref)
    torch.testing.assert_close(y.float(), ref.float(), rtol=2 ** -6, atol=3e-2)
    assert (y == ref).float().mean().item() > 0.98


def test_linear_lora_gelu():
    M, N, K = 1024, 12288, 3072
    x = _randn(M, K, seed=80)
    W = _randn(N, K, scale=1.0 / math.sqrt(K), seed=81)
    b = _randn(N, scale=0.1, seed=82)
    A = _randn(32, K, scale=1.0 / math.sqrt(K), seed=83)
    B = _randn(N, 32, scale=0.5 / math.sqrt(32), seed=84)
    y = torch.empty((M, N), dtype=torch.bfloat16, device=_dev())
    Ap, Bp = _lora_pad(A, B)
    _call_linear_lora(1, x, W, b, y, Ap, Bp, 64)
    lin = _peft_linear_ref(x, W, b, A, B)
    ref = torch.nn.functional.gelu(lin.float(), approximate="tanh").to(torch.bfloat16)
    _report("linear_lora gelu", y, ref)
    torch.testing.assert_close(y.float(), ref.float(), rtol=2 ** -6, atol=3e-2)
    assert (y == ref).float().mean().item() > 0.98


@pytest.mark.parametrize("M,heads,K,only", [(1024, 24, 3072, None), (384, 2, 256, None), (1024, 2, 256, "k")])
def test_linear_lora_qkv(M, heads, K, only):
    """stacked q|k|v with per-section adapters (only="k": a k-only adapter — q and v get a zero term)"""
    D = heads * 128
    N = 3 * D
    x = _randn(M, K, seed=90)
    W = _randn(N, K, scale=1.0 / math.sqrt(K), seed=91)
    b = _randn(N, scale=0.1, seed=92)
    nq = (1.0 + 0.1 * _randn(128, seed=93).float()).to(torch.bfloat16)
    nk = (1.0 + 0.1 * _randn(128, seed=94).float()).to(torch.bfloat16)
    cos, sin = _rope_tables(M)
    Ap = torch.zeros(192, K, dtype=torch.bfloat16, device=_dev())
    Bp = torch.zeros(N, 64, dtype=torch.bfloat16, device=_dev())
    lin = torch.empty((M, N), dtype=torch.bfloat16, device=_dev())
    for j, nm in enumerate("qkv"):
        Wj, bj = W[j * D:(j + 1) * D], b[j * D:(j + 1) * D]
        if only is None or only == nm:
            A = _randn(32, K, scale=1.0 / math.sqrt(K), seed=95 + j)
            B = _randn(D, 32, scale=0.5 / math.sqrt(32), seed=98 + j)
            Ap[64 * j:64 * j + 32] = A
            Bp[j * D:(j + 1) * D, :32] = B
            lin[:, j * D:(j + 1) * D] = _peft_linear_ref(x, Wj, bj, A, B)
        else:
            lin[:, j * D:(j + 1) * D] = _linear_ref(x, Wj, bj)
    y = torch.empty((M, N), dtype=torch.bfloat16, device=_dev())
    _call_linear_lora(3, x, W, b, y, Ap, Bp, 192, cos=cos, sin=sin, nq=nq, nk=nk)
    ref = _qkv_post_ref(lin, cos, sin, nq, nk, heads)
    _report("linear_lora qkv", y, ref)
    torch.testing.assert_close(y.float(), ref.float(), rtol=2 ** -6, atol=3e-2)


def _attn_ref(q, k, v, heads, n_main=None, mode=0, bias=0.0):
    n = q.shape[0]
    qh = q.float().view(n, heads, 128).transpose(0, 1)
    kh = k.float().view(n, heads, 128).transpose(0, 1)
    vh = v.float().view(n, heads, 128).transpose(0, 1)
    s = qh @ kh.transpose(1, 2) / math.sqrt(128.0)
    if mode:
        m = torch.zeros(n, n, device=q.device)
        val = float("-inf") if mode == 2 else bias
        m[n_main:, :n_main] = val
        m[:n_main, n_main:] = val
        s = s + m
    o = torch.softmax(s, dim=-1) @ vh
    return o.transpose(0, 1).reshape(n, heads * 128)


@pytest.mark.parametrize("n_tok,heads", [(128, 1), (256, 2), (768, 4), (200, 2), (4608, 24)])
def test_attention(n_tok, heads):
    lib = L.load()
    qkv = _randn(n_tok, 3 * heads * 128, seed=30)
    inner = heads * 128
    q, k, v = qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:]
    out = torch.full((n_tok, inner), float("nan"), dtype=torch.bfloat16, device=_dev())
    rc = lib.rf_op_attention(L.ptr(q), L.ptr(k), L.ptr(v), qkv.stride(0), L.ptr(out),
                             out.stride(0), n_tok, heads, 1, n_tok, 0, 0.0, L.cur_stream())
    L.check(rc, "rf_op_attention")
    torch.cuda.synchronize()
    ref = _attn_ref(q, k, v, heads)
    _report(f"attention n={n_tok} h={heads}", out, ref, bm=128, bn=128)
    # P is rounded to bf16 before PV and O to bf16 at the end: error ~ 2^-8 relative to |v| ~ 1
    torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=1e-2)


def test_attention_sharp_rows():
    """large score spread: the running row max jumps by > 2^8 between tiles, so the online-softmax rescale of O and the
    row sums must stay exact"""
    lib = L.load()
    n_tok, heads = 512, 2
    inner = heads * 128
    qkv = _randn(n_tok, 3 * inner, seed=31)
    qkv[:, :2 * inner] *= 4.0
    qkv[300:, inner:2 * inner] *= 3.0
    q, k, v = qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:]
    out = torch.empty((n_tok, inner), dtype=torch.bfloat16, device=_dev())
    rc = lib.rf_op_attention(L.ptr(q), L.ptr(k), L.ptr(v), qkv.stride(0), L.ptr(out),
                             out.stride(0), n_tok, heads, 1, n_tok, 0, 0.0, L.cur_stream())
    L.check(rc, "rf_op_attention")
    torch.cuda.synchronize()
    ref = _attn_ref(q, k, v, heads)
    _report("attention sharp", out, ref, bm=128, bn=128)
    torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("n_tok,n_main,heads", [(640, 512, 2), (5632, 4608, 24)])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_attention_cond_modes(mode, n_tok, n_main, heads):
    """cond-stream key ranges at the small size and at the entry-B headline geometry
    (512 txt + 4096 img + 1024 cond = 5632 tokens, 24 heads; block.py:97-125)"""
    lib = L.load()
    inner = heads * 128
    qkv = _randn(n_tok, 3 * inner, seed=32)
    q, k, v = qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:]
    bias = math.log(2.0)
    out = torch.empty((n_tok, inner), dtype=torch.bfloat16, device=_dev())
    rc = lib.rf_op_attention(L.ptr(q), L.ptr(k), L.ptr(v), qkv.stride(0), L.ptr(out),
                             out.stride(0), n_tok, heads, 1, n_main, mode, bias, L.cur_stream())
    L.check(rc, "rf_op_attention")
    torch.cuda.synchronize()
    ref = _attn_ref(q, k, v, heads, n_main, mode, bias)
    _report(f"attention cond mode {mode}", out, ref, bm=128, bn=128)
    torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=1e-2)


def test_attention_batched():
    lib = L.load()
    n_tok, heads, B = 256, 2, 3
    inner = heads * 128
    qkv = _randn(B * n_tok, 3 * inner, seed=33)
    q, k, v = qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:]
    out = torch.empty((B * n_tok, inner), dtype=torch.bfloat16, device=_dev())
    rc = lib.rf_op_attention(L.ptr(q), L.ptr(k), L.ptr(v), qkv.stride(0), L.ptr(out),
                             out.stride(0), n_tok, heads, B, n_tok, 0, 0.0, L.cur_stream())
    L.check(rc, "rf_op_attention")
    torch.cuda.synchronize()
    for b in range(B):
        sl = slice(b * n_tok, (b + 1) * n_tok)
        ref = _attn_ref(q[sl], k[sl], v[sl], heads)
        torch.testing.assert_close(out[sl].float(), ref, rtol=2e-2, atol=1e-2)


def test_ln_modulate():
    lib = L.load()
    rows, dim, B = 1000, 3072, 2
    x = _randn(rows, dim, scale=3.0, seed=40) + 0.5
    scale = _randn(B, dim, scale=0.3, seed=41)
    shift = _randn(B, dim, scale=0.3, seed=42)
    out = torch.empty_like(x)
    rc = lib.rf_op_ln_modulate(L.ptr(x), x.stride(0), L.ptr(out), out.stride(0), rows, dim,
                               L.ptr(scale), L.ptr(shift), rows // B, dim, L.cur_stream())
    L.check(rc, "rf_op_ln_modulate")
    torch.cuda.synchronize()
    ln = torch.nn.functional.layer_norm(x.float(), (dim,), eps=1e-6).to(torch.bfloat16)
    bidx = torch.arange(rows, device=_dev()) // (rows // B)
    t = (1 + scale.float()).to(torch.bfloat16)[bidx]
    u = (ln.float() * t.float()).to(torch.bfloat16)
    ref = (u.float() + shift[bidx].float()).to(torch.bfloat16)
    _report("ln_modulate", out, ref)
    torch.testing.assert_close(out.float(), ref.float(), rtol=2 ** -7, atol=2e-2)
    assert (out == ref).float().mean().item() > 0.99


@pytest.mark.parametrize("batch,N,K,act", [(1, 18432, 3072, 1), (3, 1000, 768, 0), (8, 4096, 256, 1)])
def test_gemv(batch, N, K, act):
    lib = L.load()
    x = _randn(batch, K, seed=50)
    W = _randn(N, K, scale=1.0 / math.sqrt(K), seed=51)
    b = _randn(N, seed=52)
    y = torch.empty((batch, N), dtype=torch.bfloat16, device=_dev())
    rc = lib.rf_op_gemv(L.ptr(x), x.stride(0), batch, L.ptr(W), L.ptr(b), L.ptr(y), y.stride(0), N,
                        K, act, L.cur_stream())
    L.check(rc, "rf_op_gemv")
    torch.cuda.synchronize()
    xa = torch.nn.functional.silu(x.float()).to(torch.bfloat16) if act else x
    ref = _linear_ref(xa, W, b)
    _report("gemv", y, ref)
    torch.testing.assert_close(y.float(), ref.float(), rtol=2 ** -7, atol=2e-2)


def test_timestep_embed():
    lib = L.load()
    t = torch.tensor([1.0, 0.5, 0.10473, 0.0], dtype=torch.bfloat16, device=_dev())
    out = torch.empty((4, 256), dtype=torch.bfloat16, device=_dev())
    rc = lib.rf_op_timestep_embed(L.ptr(t), 1000.0, L.ptr(out), 4, L.cur_stream())
    L.check(rc, "rf_op_timestep_embed")
    torch.cuda.synchronize()
    tv = (t * 1000).float()  # bf16 multiply like the reference
    expo = -math.log(10000) * torch.arange(128, dtype=torch.float32, device=_dev()) / 128
    arg = tv[:, None] * torch.exp(expo)[None]
    ref = torch.cat([arg.cos(), arg.sin()], -1).to(torch.bfloat16)
    _report("timestep_embed", out, ref)
    torch.testing.assert_close(out.float(), ref.float(), rtol=0, atol=2 ** -7)


def test_euler_step():
    lib = L.load()
    n = 4096 * 64
    x = _randn(n, seed=60)
    v = _randn(n, seed=61)
    sig = torch.tensor([1.0, 0.93, 0.5, 0.0], dtype=torch.float32, device=_dev())
    step = torch.tensor([1], dtype=torch.int32, device=_dev())
    ref = (x.float() + (sig[2] - sig[1]) * v.float()).to(torch.bfloat16)
    rc = lib.rf_op_euler_step(L.ptr(x), L.ptr(v), L.ptr(sig), L.ptr(step), n, L.cur_stream())
    L.check(rc, "rf_op_euler_step")
    torch.cuda.synchronize()
    assert torch.equal(x, ref)
