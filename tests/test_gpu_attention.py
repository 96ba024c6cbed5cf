"""-m gpu: the two attention kernels at the operator level, against the rounding-point references of
tests/_attn_ref.py.

  * DiT attention (csrc/attn_sm90.cu, rf_op_attention) at the headline geometries (4608 and 5632 = 4608 + 1024 tokens,
    the ragged 4544, 4544 + 576 and 4544 + 1024, 24 heads), at small edges (n = 1 ... 300, every split position class
    inside n = 300 / 384, the split inside the partial last tile, condition streams under 128 rows), biases
    bf16(log c) for c in {1.5, 2, 0.5, 1e-3}, and batch 3 in every mode.  Query rows come in four classes of
    sharpness (q scaled by 0, 1/4, 1, 3) and a block of keys past the middle is scaled by 3, so the running max moves
    late.  Bars: every element within 1 ulp_bf16(ref) + 2^-7 A (A = sum_j p_j |v_j|; tests/_attn_ref.py: within_bar
    says why not 2^-8) of the float64 kernel-order reference, and at least 99 % bit-identical in every row class of
    every fixture.
  * Invariants that need no reference and hold bit for bit by construction of the kernel, among them: cond_mode 1
    with cond_bias = -inf (generate(condition_scale=0)) is finite and equals cond_mode 2.
  * The output footprint inside a wider buffer (ld_out = 5 inner, as the single block's ACT), and the refusals.
  * Text attention (csrc/text_attn_sm90.cu) through rf_dbg_text_attention, the tensor-core path the T5 / CLIP
    encoders run: ragged S in batches, the vector and scalar bias paths, CLIP's scale and causal mask.  Bars: the same
    element bar with A = P |V| (the kernel's fp32 exp is not torch's, so a few P differ by one bf16 ulp), and at least
    99.9 % bit-identical.

Bit-identical fractions measured on one H100 80GB HBM3 (700 W power limit), lowest over the fixtures of each kind (two
runs gave the same bits):
  DiT, per row class q x 0 / 1/4 / 1 / 3:
    headline, 24 heads      0.99967 / 0.99271 / 0.99821 / 0.99929
    small edges, 1-3 heads  1.00000 / 0.99731 / 0.99894 / 0.99951
    batch 3                 0.99886 / 0.99890 / 0.99943 / 0.99978
  text: T5 0.99952, CLIP 0.99965.
The diffuse rows (q x 1/4: many keys of similar weight, so many P near rounding midpoints) sit lowest; the fp32
restatement on the CPU is lowest there too (0.996 - 0.997 at the headline sizes), the kernel a little lower because
ex2.approx is not correctly rounded.  No element was outside the element bar."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from reflectionflow_b200 import _lib as L  # noqa: E402
from tests import _attn_ref as R  # noqa: E402

DEV = "cuda:0"
NAN = float("nan")


@pytest.fixture(scope="module")
def lib():
    return R.declare(L.load())


def _attn(lib, q, k, v, n, heads, batch=1, n_main=None, mode=0, bias=0.0, out=None):
    if out is None:
        out = torch.full((batch * n, heads * 128), NAN, dtype=torch.bfloat16, device=DEV)
    rc = lib.rf_op_attention(L.ptr(q), L.ptr(k), L.ptr(v), q.stride(0), L.ptr(out), out.stride(0), n, heads, batch,
                             n if n_main is None else n_main, mode, bias, L.cur_stream())
    L.check(rc, "rf_op_attention")
    torch.cuda.synchronize()
    return out


def _operands(n, heads, batch=1, seed=0):
    return R.split_qkv(R.dit_operands(n, heads, batch, seed, DEV), heads)


# ------------------------------------------------------------------------------------ DiT: against the reference
@pytest.mark.parametrize("name", list(R.DIT_FIXTURES))
def test_dit_attention_matches_the_kernel_order_reference(lib, name):
    q, k, v, n, heads, batch, n_main, mode, bias = R.dit_fixture(name, DEV)
    out = _attn(lib, q, k, v, n, heads, batch, n_main, mode, bias)
    ref, A = R.dit_attention(q, k, v, heads, n, batch, n_main, mode, bias)
    rows = torch.arange(n)
    ok, fr = R.dit_check(out, ref, A, rows, heads, batch)
    bad = ~(R.within_bar(out, ref, A) & torch.isfinite(out.float()))
    print(f"[{name}] identical per row class " + " ".join(f"{c}:{f:.5f}" for c, f in fr.items()) +
          f" ; outside the bar {int(bad.sum())}")
    if bad.any():
        r, c = bad.nonzero()[0].tolist()
        print(f"  first at row {r} col {c}: got {out[r, c].item()} ref {ref[r, c].item()} A {A[r, c].item():.4g}")
    assert ok
    assert min(fr.values()) >= R.DIT_IDENTICAL


# ------------------------------------------------------------------------------------ DiT: invariants
# (n_tok, n_main, heads): tile-aligned split, the 4544 + 1024 headline split (inside a tile, then a tail), a small
# ragged split and a split inside the partial last tile
GEOMS = [(640, 512, 2), (5568, 4544, 2), (300, 77, 3), (300, 290, 2)]


@pytest.mark.parametrize("n,n_main,heads", GEOMS)
def test_cond_bias_zero_equals_plain_attention(lib, n, n_main, heads):
    q, k, v = _operands(n, heads, seed=n + n_main)
    assert torch.equal(_attn(lib, q, k, v, n, heads, 1, n_main, 1, 0.0), _attn(lib, q, k, v, n, heads))


@pytest.mark.parametrize("n,n_main,heads", GEOMS + [(5632, 4608, 24)])
def test_cond_bias_minus_inf_is_the_union_mask(lib, n, n_main, heads):
    """condition_scale = 0: the reference's bias log 0 = -inf gives the cross pairs weight 0, exactly the
    union_cond_attn = False mask"""
    q, k, v = _operands(n, heads, seed=n + n_main + 1)
    got = _attn(lib, q, k, v, n, heads, 1, n_main, 1, float("-inf"))
    assert torch.isfinite(got.float()).all(), f"{int((~torch.isfinite(got.float())).any(1).sum())} rows not finite"
    assert torch.equal(got, _attn(lib, q, k, v, n, heads, 1, n_main, 2))


@pytest.mark.parametrize("n,n_main,heads", GEOMS)
def test_masked_main_rows_equal_the_main_tokens_alone(lib, n, n_main, heads):
    """cond_mode 2: the main rows walk the main keys, then fully masked condition tiles that leave m, l and O as they
    are (ex2.approx(0) == 1): the same bits as a plain call over the main tokens"""
    q, k, v = _operands(n, heads, seed=n + n_main + 2)
    got = _attn(lib, q, k, v, n, heads, 1, n_main, 2)
    alone = _attn(lib, q[:n_main], k[:n_main], v[:n_main], n_main, heads)
    assert torch.equal(got[:n_main], alone)


@pytest.mark.parametrize("n,n_main,heads", [(640, 512, 2), (5632, 4608, 2), (384, 128, 1)])
def test_masked_condition_rows_equal_the_condition_tokens_alone(lib, n, n_main, heads):
    """cond_mode 2 with n_main % 128 == 0: the condition rows skip every main tile"""
    q, k, v = _operands(n, heads, seed=n + n_main + 3)
    got = _attn(lib, q, k, v, n, heads, 1, n_main, 2)
    alone = _attn(lib, q[n_main:], k[n_main:], v[n_main:], n - n_main, heads)
    assert torch.equal(got[n_main:], alone)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("n,n_main", [(256, 200), (384, 256)])
def test_batch_equals_single_calls(lib, n, n_main, mode):
    heads, B = 2, 3
    q, k, v = _operands(n, heads, B, seed=n + mode)
    bias = R.cond_bias(2.0)
    got = _attn(lib, q, k, v, n, heads, B, n_main, mode, bias)
    for b in range(B):
        r = slice(b * n, (b + 1) * n)
        assert torch.equal(got[r], _attn(lib, q[r], k[r], v[r], n, heads, 1, n_main, mode, bias)), b


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_heads_are_independent(lib, mode):
    n, n_main, heads = 5568, 4544, 3
    q, k, v = _operands(n, heads, seed=7 + mode)
    bias = R.cond_bias(0.5)
    got = _attn(lib, q, k, v, n, heads, 1, n_main, mode, bias)
    for h in range(heads):
        others = torch.ones(heads * 128, dtype=torch.bool, device=DEV)
        others[h * 128:(h + 1) * 128] = False
        q2, k2, v2 = q.clone(), k.clone(), v.clone()
        for t in (q2, k2, v2):
            t[:, others] = -t[:, others] * 2
        got2 = _attn(lib, q2, k2, v2, n, heads, 1, n_main, mode, bias)
        cols = slice(h * 128, (h + 1) * 128)
        assert torch.equal(got2[:, cols], got[:, cols]), h


def test_two_runs_are_identical(lib):
    n, n_main, heads = 5568, 4544, 24
    q, k, v = _operands(n, heads, seed=11)
    bias = R.cond_bias(2.0)
    assert torch.equal(_attn(lib, q, k, v, n, heads, 1, n_main, 1, bias),
                       _attn(lib, q, k, v, n, heads, 1, n_main, 1, bias))


# ------------------------------------------------------------------------------------ DiT: footprint, refusals
@pytest.mark.parametrize("n,heads,batch,n_main,mode", [(4544, 24, 1, None, 0), (300, 3, 1, 77, 1), (256, 2, 3, 200, 2),
                                                       (5568, 24, 1, 4544, 2)])
def test_output_footprint_in_a_wider_buffer(lib, n, heads, batch, n_main, mode):
    """dit.cu writes the single block's attention into ACT[:, 0:D] with ld_out = 5 D, next to the MLP hidden in
    ACT[:, D:5D]: columns >= inner and rows >= batch n_tok stay untouched, and the bits equal the ld_out = inner run"""
    inner = heads * 128
    q, k, v = _operands(n, heads, batch, seed=n + heads)
    bias = R.cond_bias(1.5)
    buf = torch.full((batch * n + 16, 5 * inner), -3.25, dtype=torch.bfloat16, device=DEV)
    before = buf.clone()
    _attn(lib, q, k, v, n, heads, batch, n_main, mode, bias, out=buf[:batch * n, :inner])
    tight = _attn(lib, q, k, v, n, heads, batch, n_main, mode, bias)
    assert torch.equal(buf[:, inner:], before[:, inner:])
    assert torch.equal(buf[batch * n:], before[batch * n:])
    assert torch.equal(buf[:batch * n, :inner], tight)


def _refused(lib, n, heads, batch, n_main, mode, ld_out, match):
    q, k, v = _operands(n, heads, batch)
    out = torch.zeros(batch * n, 5 * heads * 128, dtype=torch.bfloat16, device=DEV)
    rc = lib.rf_op_attention(L.ptr(q), L.ptr(k), L.ptr(v), q.stride(0), L.ptr(out), ld_out, n, heads, batch, n_main,
                             mode, 0.5, L.cur_stream())
    torch.cuda.synchronize()
    assert rc != 0 and match in lib.rf_last_error().decode()
    assert not out.any()


@pytest.mark.parametrize("n_main", [0, -5, 300, 301])
@pytest.mark.parametrize("mode", [1, 2])
def test_refuses_a_split_outside_the_sequence(lib, n_main, mode):
    _refused(lib, 300, 1, 1, n_main, mode, 128, "cond split must lie inside")


def test_refuses_a_ragged_batch(lib):
    _refused(lib, 300, 1, 2, 300, 0, 128, "n_tok % 128 == 0")


def test_refuses_an_odd_output_pitch(lib):
    _refused(lib, 256, 1, 1, 256, 0, 129, "4-byte aligned")


# ------------------------------------------------------------------------------------ text attention
def _text(lib, q, k, v, B, S, heads, bias, scale, use_scale, causal, out=None):
    if out is None:
        out = torch.full((B * S, heads * 64), NAN, dtype=torch.bfloat16, device=DEV)
    rc = lib.rf_dbg_text_attention(L.ptr(q), L.ptr(k), L.ptr(v), q.stride(0), L.ptr(out), out.stride(0), B, S, heads,
                                   L.ptr(bias), scale, use_scale, causal, L.cur_stream())
    L.check(rc, "rf_dbg_text_attention")
    torch.cuda.synchronize()
    return out


def _text_fixture(name):
    B, S, heads, kind, off = R.TEXT_FIXTURES[name]
    qkv, bias = R.text_operands(B, S, heads, kind, off, R.seed_of(name), DEV)
    inner = heads * 64
    return (qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:], B, S, heads, bias) + R.text_args(kind)


@pytest.mark.parametrize("name", list(R.TEXT_FIXTURES))
def test_text_attention_matches_the_eager_rounding_points(lib, name):
    args = _text_fixture(name)
    out = _text(lib, *args).float()
    ref, A = R.text_attention(*args)
    same = (out == ref).double().mean().item()
    bad = ~(R.within_bar(out, ref, A) & torch.isfinite(out))
    print(f"[{name}] identical {same:.5f} ; outside the bar {int(bad.sum())}")
    if bad.any():
        r, c = bad.nonzero()[0].tolist()
        print(f"  first at row {r} col {c}: got {out[r, c].item()} ref {ref[r, c].item()}")
    assert not bad.any()
    assert same >= R.TEXT_IDENTICAL


@pytest.mark.parametrize("name", ["t5_S300_h4_B3", "t5_S512_h1_B3", "clip_S77_h4_B3"])
def test_text_output_footprint_in_a_wider_buffer(lib, name):
    q, k, v, B, S, heads, bias, scale, use_scale, causal = _text_fixture(name)
    inner = heads * 64
    buf = torch.full((B * S + 16, 5 * inner), -3.25, dtype=torch.bfloat16, device=DEV)
    before = buf.clone()
    _text(lib, q, k, v, B, S, heads, bias, scale, use_scale, causal, out=buf[:B * S, :inner])
    tight = _text(lib, q, k, v, B, S, heads, bias, scale, use_scale, causal)
    assert torch.equal(buf[:, inner:], before[:, inner:])
    assert torch.equal(buf[B * S:], before[B * S:])
    assert torch.equal(buf[:B * S, :inner], tight)


def test_text_hook_refuses_what_the_tensor_core_path_does_not_take(lib):
    q = torch.zeros(513, 3 * 64, dtype=torch.bfloat16, device=DEV)
    out = torch.zeros(513, 64, dtype=torch.bfloat16, device=DEV)
    rc = lib.rf_dbg_text_attention(L.ptr(q), L.ptr(q), L.ptr(q), q.stride(0), L.ptr(out), 64, 1, 513, 1, None, 1.0,
                                   0, 0, L.cur_stream())
    assert rc != 0 and "S <= 512" in lib.rf_last_error().decode()


# ------------------------------------------------------------------------------------ model level
@pytest.mark.parametrize("n_txt,cond_side", [(128, 8), (77, 16)])
def test_generate_condition_scale_zero_is_the_union_mask(n_txt, cond_side):
    """generate(condition_scale=0): the reference's c_factor bias is log 0 = -inf on the cross blocks (block.py:115-122),
    and SDPA then computes what the union_cond_attn = False mask gives.  n_txt 128 + 256 image tokens puts the split on
    a tile edge; 77 + 256 puts it inside a tile."""
    from reflectionflow_b200.config import FluxDiTConfig
    from reflectionflow_b200.pipeline import B200FluxPipeline, Condition, generate
    pipe = B200FluxPipeline.from_synthetic(FluxDiTConfig(num_layers=1, num_single_layers=1), seed=0)
    g = torch.Generator().manual_seed(n_txt)
    pe = torch.randn(1, n_txt, 4096, generator=g).to(torch.bfloat16).to(DEV)
    pooled = torch.randn(1, 768, generator=g).to(torch.bfloat16).to(DEV)
    cond = torch.randn(1, cond_side * cond_side, 64, generator=g).to(torch.bfloat16)

    def run(condition_scale, model_config):
        return generate(pipe, conditions=[Condition("cot", latents=cond)], model_config=model_config,
                        condition_scale=condition_scale, default_lora=True, prompt_embeds=pe,
                        pooled_prompt_embeds=pooled, height=256, width=256, num_inference_steps=2,
                        output_type="latent", generator=torch.Generator("cpu").manual_seed(0)).images.clone()

    zero = run(0.0, {})
    masked = run(1.0, {"union_cond_attn": False})
    pipe.transformer.close()
    assert torch.isfinite(zero.float()).all()
    assert torch.equal(zero, masked)
