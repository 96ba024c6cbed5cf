"""-m gpu: the text encoders' own kernels one launch at a time through the rf_dbg_text_* / rf_dbg_t5_gated_gelu hooks
(csrc/rf_api.cu), which call the launchers rf_t5_encode / rf_clip_encode run.  The oracles are transformers' modules and
torch ops run on the device in bf16, as the reference runs them, plus the restatements of tests/_text_ref.py.

  * T5's gated half (wi_0 GEMM, wi_1 GEMM, gelu_new product): bit-exact against NewGELUActivation(bf16(x wi_0^T)) *
    bf16(x wi_1^T) on exact operands (_exact.py's grids, so both GEMM outputs are known exactly).  On random operands
    at T5-XXL width, wi_1 x at test_gpu_ops.py's GEMM bars, and each product NewGELUActivation of a value within 2 ulps
    of bf16(x wi_0^T), times the kernel's h1, or within those bars.
  * The activations: every finite bf16 value through gelu_new (b = 1) and quick-GELU, bit-exact against the device's
    NewGELUActivation / QuickGELUActivation; 1 M random products, in place and not; a partial last block.
  * T5LayerNorm / LayerNorm at the encoders' eps, one bf16 ulp at the rounding points: T5LayerNorm's output is
    bf16(w h') with h' within 1 ulp of its normalised value h on the device (its second rounding can turn that ulp
    into two of the output); LayerNorm's within 1 ulp of F.layer_norm on the device or of the float64 truth rounded
    once, widened where t w and b cancel or the row sits far from 0 (as in test_gpu_vae_ops.py's GroupNorm).  At most
    0.1 % of each case's elements (at least one) bit-identical to neither; 1 % for LayerNorm rows at mean / std = 128,
    where both fp32 implementations lose bits to the offset.  Rows are not multiples of the 8 a block covers.
  * Embedding gathers (T5 at d 4096 over the whole vocabulary's range, CLIP with positions) and the pooled-row gather:
    bit-exact.  Every output buffer carries a sentinel guard that must come back untouched.
  * Token ids outside the vocabulary are refused by B200TextEncoders before any launch.

Measured on one H100 80GB HBM3 (700 W power limit):
  gated half, exact operands      bit-exact at all 12 shapes; with the fused GELU-tanh epilogue the encoder used before,
                                  0.41 to 0.45 of the products differ
  gated half, random operands     all within the bar; 0.9980 bit-identical at T5-XXL width (512 x 4096 x 10240)
  gelu_new, quick-GELU            0 differences on all 65280 finite bf16 values; the restatements equal the device too
  products, 1 M random pairs      bit-exact, in place and not
  T5LayerNorm                     max 2 ulps of the output, all within the bar; lowest bit-identical fraction 0.999956
  LayerNorm                       all within the bar; lowest bit-identical fraction 0.99972 (0.9951 identical to torch
                                  or the truth at mean / std = 128, where torch alone matches the truth on 0.9851)
  embeddings, gather              bit-exact"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from reflectionflow_b200 import _lib as L  # noqa: E402
from tests import _exact as E  # noqa: E402
from tests import _text_ref as R  # noqa: E402

DEV = "cuda:0"
BF = torch.bfloat16
SENT = 0x7FA5  # a NaN bit pattern no kernel writes: every element a launch must not touch holds it
GUARD = 4096


@pytest.fixture(scope="module")
def lib():
    return R.declare(L.load())


def _s():
    return L.cur_stream()


def _buf(n):
    t = torch.empty(n + GUARD, dtype=BF, device=DEV)
    t.view(torch.int16).fill_(SENT)
    return t


def _untouched(buf, n):
    assert bool((buf[n:].view(torch.int16) == SENT).all()), "write past the end of the output"


def _bits_eq(got, ref):
    return got.to(BF).view(torch.int16) == ref.to(BF).view(torch.int16)


def _ndiff(got, ref):
    return int((~_bits_eq(got, ref)).sum())


def _step(t, k):
    """the bf16 value k steps from t along the bf16 number line"""
    b = t.to(BF).view(torch.int16).int()
    line = torch.where(b < 0, -(b & 0x7FFF), b) + k
    return torch.where(line < 0, (-line) | 0x8000, line).to(torch.int16).view(BF).float()


def _new_gelu(x):
    from transformers.activations import NewGELUActivation
    return NewGELUActivation()(x)


def _quick_gelu(x):
    from transformers.activations import QuickGELUActivation
    return QuickGELUActivation()(x)


# ------------------------------------------------------------------------------------ T5's gated half
def _gated(lib, x, wi0, wi1):
    T, D = x.shape
    Fd = wi0.shape[0]
    h0, h1 = _buf(T * Fd), _buf(T * Fd)
    L.check(lib.rf_dbg_t5_gated_gelu(R.ptr(x), T, D, R.ptr(wi0), R.ptr(wi1), Fd, R.ptr(h0), R.ptr(h1), _s()),
            "rf_dbg_t5_gated_gelu")
    torch.cuda.synchronize()
    _untouched(h0, T * Fd)
    _untouched(h1, T * Fd)
    return h0[:T * Fd].view(T, Fd), h1[:T * Fd].view(T, Fd)


@pytest.mark.parametrize("Fd", [512, 2560])
@pytest.mark.parametrize("D", [256, 1024])
@pytest.mark.parametrize("T", [77, 231, 512])
def test_gated_half_exact_operands(lib, T, D, Fd):
    seed = T * 31 + D * 7 + Fd
    x = E.act((T, D), seed).to(DEV)
    wi0 = E.weight((Fd, D), seed + 1).to(DEV)
    wi1 = E.weight((Fd, D), seed + 2).to(DEV)
    a = E.bf(E.gemm(x, wi0)).to(BF)  # exact accumulators: the only rounding is the bf16 one
    b = E.bf(E.gemm(x, wi1)).to(BF)
    h0, h1 = _gated(lib, x, wi0, wi1)
    assert _ndiff(h1, b) == 0, "wi_1 GEMM"
    want = _new_gelu(a) * b  # T5DenseGatedActDense in bf16 on the device
    bad = _ndiff(h0, want)
    print(f"[gated T {T} D {D} F {Fd}] {bad} of {want.numel()} ({bad / want.numel():.4f}) differ from "
          f"NewGELUActivation(h0) * h1")
    assert bad == 0, f"{bad} of {want.numel()} ({bad / want.numel():.4f}) products differ"


@pytest.mark.parametrize("T,D,Fd", [(77, 1024, 2560), (512, 4096, 10240)])
def test_gated_half_random_operands(lib, T, D, Fd):
    x = E.randn((T, D), T + D).to(DEV)
    wi0 = E.randn((Fd, D), T + D + 1, D ** -0.5).to(DEV)
    wi1 = E.randn((Fd, D), T + D + 2, D ** -0.5).to(DEV)
    h0, h1 = _gated(lib, x, wi0, wi1)
    a = E.bf(E.gemm(x, wi0, exact=False))
    b = E.bf(E.gemm(x, wi1, exact=False)).to(BF)
    torch.testing.assert_close(h1.float(), b.float(), rtol=2 ** -7, atol=2e-2)
    # the fp32 sums of wi_0 x land on the other side of a bf16 midpoint now and then, and gelu_new's chain turns one
    # ulp of its input into several ulps of its output where 1 + tanh cancels: each product must be the device's
    # NewGELUActivation of a value within 2 ulps of bf16(x wi_0^T), times the kernel's own h1, or within the GEMM bars
    want = _new_gelu(a.to(BF)) * h1
    ok = torch.isclose(h0.float(), want.float(), rtol=2 ** -7, atol=2e-2)
    for k in (-2, -1, 1, 2):
        ok |= _bits_eq(h0, _new_gelu(_step(a, k).to(BF)) * h1)
    same = 1 - _ndiff(h0, want) / want.numel()
    print(f"[gated random T {T} D {D} F {Fd}] outside the bar {int((~ok).sum())}, bit-identical {same:.5f}")
    assert bool(ok.all())


# ------------------------------------------------------------------------------------ activations
def _ewise(lib, a, b, mode, inplace=False):
    n = a.numel()
    if inplace:
        out = _buf(n)
        out[:n] = a
        src = out
    else:
        out, src = _buf(n), a
    L.check(lib.rf_dbg_text_ewise(R.ptr(src), R.ptr(b), R.ptr(out), n, mode, _s()), "rf_dbg_text_ewise")
    torch.cuda.synchronize()
    _untouched(out, n)
    return out[:n]


def _report(tag, x, got, want):
    bad = got.to(BF).view(torch.int16) != want.to(BF).view(torch.int16)
    first = [(float(x[i]), float(got[i]), float(want[i])) for i in bad.nonzero().flatten()[:8].tolist()]
    print(f"[{tag}] {int(bad.sum())} of {x.numel()} differ; first (x, ours, torch): {first}")
    return int(bad.sum())


def test_gelu_new_every_bf16_value(lib):
    v = R.all_finite_bf16().to(DEV)  # 65280 = 8 x 8160 elements: the last block of 256 threads is partial
    got = _ewise(lib, v, torch.ones_like(v), 0)
    want = _new_gelu(v)
    assert _report("gelu_new vs NewGELUActivation", v, got, want) == 0
    assert _report("restatement vs NewGELUActivation", v, R.gelu_new(v), want) == 0


def test_quick_gelu_every_bf16_value(lib):
    v = R.all_finite_bf16().to(DEV)
    got = _ewise(lib, v, None, 1)
    want = _quick_gelu(v)
    assert _report("quick_gelu vs QuickGELUActivation", v, got, want) == 0
    assert _report("restatement vs QuickGELUActivation", v, R.quick_gelu(v), want) == 0


@pytest.mark.parametrize("inplace", [False, True])
def test_gated_product_random_pairs(lib, inplace):
    a, b = (t.to(DEV) for t in R.random_pairs())
    got = _ewise(lib, a, b, 0, inplace)
    assert _report(f"product, in place {inplace}", a, got, _new_gelu(a) * b) == 0
    assert _ndiff(got, R.gated(a, b)) == 0


@pytest.mark.parametrize("mode", [0, 1])
def test_ewise_partial_last_block(lib, mode):
    n = 8 * (256 * 3 + 37)
    a, b = (t[:n].to(DEV) for t in R.random_pairs(seed=5))
    got = _ewise(lib, a, b if mode == 0 else None, mode, inplace=True)
    want = _new_gelu(a) * b if mode == 0 else _quick_gelu(a)
    assert _ndiff(got, want) == 0


def test_ewise_refuses_ragged_counts(lib):
    z = torch.zeros(16, dtype=BF, device=DEV)
    assert lib.rf_dbg_text_ewise(R.ptr(z), R.ptr(z), R.ptr(z), 12, 0, _s()) == -1
    assert lib.rf_dbg_text_ewise(R.ptr(z), None, R.ptr(z), 16, 0, _s()) == -1


# ------------------------------------------------------------------------------------ row norms
NORM_FMA_SLACK = 2.0 ** -20  # 8 fp32 ulps of the summands of LayerNorm's last step, where they cancel
NORM_IDENTICAL = 0.001  # at most this fraction of a case's elements (and at least one) not bit-identical
# ... except LayerNorm rows at mean / std = 128: there the fp32 means of F.layer_norm on the device and of the kernel are
# both off by a few 1e-6, which moves outputs near 0.  Measured: F.layer_norm differs from the float64 truth on up to
# 1.5 % of them, the kernel on up to 1.0 %, and up to 0.49 % of the kernel's outputs equal neither
NORM_IDENTICAL_OFFSET = 0.01


def _torch_norm(x, w, b, mode):
    if mode == 0:
        from transformers.models.t5.modeling_t5 import T5LayerNorm
        m = T5LayerNorm(x.shape[1], eps=R.T5_EPS).to(DEV, BF)
        with torch.no_grad():
            m.weight.copy_(w)
            return m(x)
    with torch.no_grad():
        return F.layer_norm(x, (x.shape[1],), w, b, R.CLIP_EPS)


def _rms_check(got, x, w, want):
    """T5LayerNorm rounds twice: h = bf16(x rsqrt(var + eps)), then bf16(w h).  The kernel's 1 / sqrt and fp32 sum
    order move h by at most one ulp, which w h can turn into two ulps of the output where it drops a binade: each
    output must be bf16(w h') for h' within one ulp of the device's own h."""
    xf = x.float()
    h = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + R.T5_EPS)).to(BF)
    assert _ndiff(w * h, want) == 0  # h is T5LayerNorm's rounding point
    ok = torch.zeros_like(got, dtype=torch.bool)
    for k in (-1, 0, 1):
        ok |= _bits_eq(got, E.bf(w.float() * _step(h, k)))
    return ok, ~_bits_eq(got, want)


def _ln_check(got, x, w, b, want):
    """one rounding of (x - mean) rstd w + b: within one ulp of F.layer_norm on the device or of the float64 truth
    rounded once (their fp32 statistics differ), widened where t w and b cancel or the row sits far from 0 (an fp32
    mean of values near 128 is off by ~1e-5); bit-identical to one of the two."""
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + R.CLIP_EPS)
    terms = ((xd - mean) * rstd * w.double()).abs() + b.double().abs() + (mean * rstd * w.double()).abs()
    truth = R.layer_norm(x, w, b)

    def near(ref):
        return (E.ulps(got, ref) <= 1) | ((got.double() - ref.double()).abs() <= NORM_FMA_SLACK * terms)

    return near(want) | near(truth), ~_bits_eq(got, want) & ~_bits_eq(got, truth)


@pytest.mark.parametrize("rows", R.NORM_ROWS)
@pytest.mark.parametrize("dim", R.NORM_DIMS)
@pytest.mark.parametrize("mode", [0, 1])
def test_rownorm(lib, mode, dim, rows):
    eps = R.T5_EPS if mode == 0 else R.CLIP_EPS
    for case in R.NORM_CASES[mode]:
        x, w, b = (None if t is None else t.to(DEV) for t in R.norm_inputs(rows, dim, case, mode))
        out = _buf(rows * dim)
        L.check(lib.rf_dbg_text_rownorm(R.ptr(x), R.ptr(out), rows, dim, R.ptr(w), R.ptr(b), eps, mode, _s()),
                "rf_dbg_text_rownorm")
        torch.cuda.synchronize()
        _untouched(out, rows * dim)
        got = out[:rows * dim].view(rows, dim)
        want = _torch_norm(x, w, b, mode)
        ok, differs = _rms_check(got, x, w, want) if mode == 0 else _ln_check(got, x, w, b, want)
        n = got.numel()
        ref = R.t5_layernorm(x, w) if mode == 0 else R.layer_norm(x, w, b)
        print(f"[{'rms' if mode == 0 else 'ln'} {rows}x{dim} {case}] max ulps vs torch {int(E.ulps(got, want).max())} "
              f"outside bar {int((~ok).sum())}; bit-identical to torch {1 - _ndiff(got, want) / n:.6f}, to the "
              f"restatement {1 - _ndiff(got, ref) / n:.6f}, to neither {int(differs.sum())}; torch vs restatement "
              f"{1 - _ndiff(want, ref) / n:.6f}")
        assert torch.isfinite(got.float()).all()
        assert bool(ok.all()), case
        assert int(differs.sum()) <= max(1, int((NORM_IDENTICAL_OFFSET if case == "offset" else NORM_IDENTICAL) * n)), case
        if case == "zero_row":
            z = got[rows // 2].float()
            assert bool((z == 0).all()) if mode == 0 else _ndiff(z, b) == 0


# ------------------------------------------------------------------------------------ embeddings and gathers
def _embed(lib, ids, table, pos, S):
    T, D = ids.numel(), table.shape[1]
    ids32 = ids.to(DEV, torch.int32).contiguous()
    out = _buf(T * D)
    L.check(lib.rf_dbg_text_embed(R.ptr(ids32), R.ptr(table), R.ptr(pos), R.ptr(out), T, S, D, _s()),
            "rf_dbg_text_embed")
    torch.cuda.synchronize()
    _untouched(out, T * D)
    return out[:T * D].view(T, D)


def test_t5_embed_whole_vocabulary(lib):
    vocab, D, B, S = 32128, 4096, 3, 77
    g = torch.Generator(device=DEV).manual_seed(0)
    table = torch.randn(vocab, D, generator=g, device=DEV).to(BF)
    ids = torch.randint(0, vocab, (B, S), generator=torch.Generator().manual_seed(1))
    ids[0, 0], ids[0, -1], ids[1, 3], ids[2, -1] = 0, vocab - 1, vocab - 1, 0
    got = _embed(lib, ids.flatten(), table, None, S)
    assert _ndiff(got, F.embedding(ids.flatten().to(DEV), table)) == 0


@pytest.mark.parametrize("S", [20, 77])
def test_clip_embed_with_positions(lib, S):
    from transformers import CLIPTextConfig
    from transformers.models.clip.modeling_clip import CLIPTextEmbeddings
    vocab, C, B = 49408, 768, 3
    m = CLIPTextEmbeddings(CLIPTextConfig(vocab_size=vocab, hidden_size=768, max_position_embeddings=77))
    g = torch.Generator().manual_seed(S)
    with torch.no_grad():
        m.token_embedding.weight.copy_(torch.randn(vocab, C, generator=g) * 0.5)
        m.position_embedding.weight.copy_(torch.randn(77, C, generator=g) * 0.5)
    m = m.to(DEV, BF)
    ids = torch.randint(0, vocab, (B, S), generator=g)
    ids[0, 0], ids[1, -1], ids[2, S // 2] = 0, vocab - 1, vocab - 1
    table, pos = m.token_embedding.weight.detach(), m.position_embedding.weight.detach()
    got = _embed(lib, ids.flatten(), table, pos, S)
    with torch.no_grad():
        want = m(input_ids=ids.to(DEV)).reshape(B * S, C)
    assert _ndiff(got, want) == 0
    assert _ndiff(got, R.embed(ids.flatten().to(DEV), table, pos, S)) == 0


@pytest.mark.parametrize("S,D", [(20, 768), (77, 768), (77, 4096)])
def test_gather_rows(lib, S, D):
    B = 3
    x = E.randn((B * S, D), S + D, device=DEV)
    pos = torch.tensor([0, S - 1, S // 2], dtype=torch.int32, device=DEV)
    out = _buf(B * D)
    L.check(lib.rf_dbg_text_gather_rows(R.ptr(x), R.ptr(pos), R.ptr(out), B, S, D, _s()), "rf_dbg_text_gather_rows")
    torch.cuda.synchronize()
    _untouched(out, B * D)
    assert _ndiff(out[:B * D].view(B, D), R.gather(x, pos, S)) == 0


# ------------------------------------------------------------------------------------ token ids out of range
_ENC = {}


def _encoders():
    if not _ENC:
        from reflectionflow_b200.text import B200TextEncoders
        _ENC["e"] = B200TextEncoders(t5_layers=1, t5_d_model=256, t5_d_ff=512, t5_heads=4, t5_vocab=64, clip_layers=1,
                                     clip_d_model=256, clip_heads=4, clip_vocab=64,
                                     clip_max_pos=77).init_synthetic_weights(seed=0)
    return _ENC["e"]


@pytest.mark.parametrize("bad", [-1, 64, 1 << 20])
@pytest.mark.parametrize("which", ["t5", "clip"])
def test_token_ids_outside_the_vocabulary_are_refused(which, bad):
    enc = _encoders()
    run = enc.t5_encode if which == "t5" else enc.clip_encode
    lib = L.load()
    ids = torch.randint(0, 64, (2, 20), generator=torch.Generator().manual_seed(2))
    n0 = lib.rf_launch_count()
    run(ids)
    torch.cuda.synchronize()
    assert lib.rf_launch_count() > n0  # the valid ids run
    ids[1, 7] = bad
    n0 = lib.rf_launch_count()
    with pytest.raises(L.RFError, match="token id outside"):
        run(ids)
    assert lib.rf_launch_count() == n0, "a kernel was launched with an id outside the vocabulary"
