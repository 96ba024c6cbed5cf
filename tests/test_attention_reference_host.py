"""-m "not gpu": the attention references of tests/_attn_ref.py, on the CPU, at CPU-sized cuts of the fixtures the GPU
tests run (the first one or two heads, the query rows of tests/_attn_ref.py: probe_rows).

  * The bars of tests/test_gpu_attention.py are reachable by fp32 arithmetic: the kernel's order restated in fp32
    passes them against the float64 reference.
  * The bars can fail: each reference with one deliberate change (tests/_attn_ref.py: MUTATIONS) fails them on at
    least one fixture the GPU tests also run.
  * The text reference is the eager sequence: torch's own CPU bf16 ops (matmul, add, softmax(float), matmul) give the
    same probabilities bit for bit, and outputs within the text bars (torch accumulates P V in fp32, in its own order)."""
import functools

import pytest
import torch

from tests import _attn_ref as R

HOST_DIT = ("n4608", "n4544", "n5568_m1", "n5568_m2", "n384_s129_m1", "n384_s1_m2", "n300_s290_m1",
            "n300_s290_m2", "n300_s77_m1", "b3_n256_m1", "b3_n384_m2", "n129", "n1")
HOST_TEXT = ("t5_S77_h4_B1", "t5_S300_h4_B3", "t5_S129_h1_B3", "t5_S256_h4_B1_off2", "t5_S512_h4_B3_off2",
             "clip_S77_h4_B3", "clip_S300_h4_B3")


@functools.lru_cache(maxsize=None)
def _dit(name):
    q, k, v, n, heads, batch, n_main, mode, bias = R.dit_fixture(name)
    rows = R.probe_rows(n, n_main)
    args = (q, k, v, min(heads, 2), n, batch, n_main, mode, bias)
    ref, A = R.dit_attention(*args, rows=rows)
    return args, rows, ref, A


@pytest.mark.parametrize("name", HOST_DIT)
def test_dit_fp32_restatement_passes_the_bars(name):
    args, rows, ref, A = _dit(name)
    got, _ = R.dit_attention(*args, rows=rows, dtype=torch.float32)
    ok, fr = R.dit_check(got, ref, A, rows, args[3], args[5])
    print(f"[{name}] fp32 restatement: identical per row class " + " ".join(f"{c}:{f:.4f}" for c, f in fr.items()))
    assert ok and min(fr.values()) >= R.DIT_IDENTICAL


@pytest.mark.parametrize("mut", R.DIT_MUTATIONS)
def test_dit_mutation_fails_the_bars(mut):
    caught = []
    for name in HOST_DIT:
        args, rows, ref, A = _dit(name)
        bad, _ = R.dit_attention(*args, rows=rows, mut=(mut,))
        if not R.dit_passes(bad, ref, A, rows, args[3], args[5]):
            caught.append(name)
    print(f"{R.MUTATIONS[mut]}: fails the bars on {caught}")
    assert caught


@pytest.mark.parametrize("name", ("n300_s77_m1", "n5568_m2", "b3_n256_m1"))
def test_dit_reference_is_within_the_bar_of_the_plain_softmax(name):
    """the kernel-order reference and the plain float64 softmax differ by the P rounding only: within the bar"""
    (q, k, v, heads, n, batch, n_main, mode, bias), rows, ref, A = _dit(name)
    plain = R.dit_plain(q, k, v, heads, n, batch, n_main, mode, bias)
    idx = torch.cat([b * n + rows for b in range(batch)])
    assert bool(R.within_bar(plain[idx], ref, A).all())


def test_dit_bar_needs_2_to_the_minus_7():
    """the element bar's 2^-7 A: on a sharp row whose second-largest weight is 0.568 (v = -1.92), the fp32 restatement
    rounds that P to the other side of a midpoint and lands 2 ulps (0.0078) from the float64 reference, beyond
    1 ulp + 2^-8 A (0.0077) but within 1 ulp + 2^-7 A"""
    q, k, v, n, heads, batch, n_main, mode, bias = R.dit_fixture("n5568_m1")
    cs, rows = slice(128, 256), torch.tensor([1803])
    args = (q[:, cs], k[:, cs], v[:, cs], 1, n, 1, n_main, mode, bias)
    ref, A = R.dit_attention(*args, rows=rows)
    got, _ = R.dit_attention(*args, rows=rows, dtype=torch.float32)
    d, ulp, a = (got - ref)[0, 32].abs().item(), R.ulp_bf16(ref)[0, 32].item(), A[0, 32].item()
    assert ulp + 2.0 ** -8 * a < d <= ulp + 2.0 ** -7 * a


def test_dit_uniform_rows_are_the_mean_of_v():
    """rows with q = 0 (class 0) see equal scores: P = 1 in every tile, so the reference is bf16(mean of the
    unmasked V rows), whatever the tiling"""
    (q, k, v, heads, n, batch, n_main, mode, bias), rows, ref, A = _dit("n4544")
    sel = rows % 4 == 0
    mean = v[:n, :heads * 128].double().mean(dim=0)
    assert torch.equal(ref[sel], R.bf(mean).expand(int(sel.sum()), -1))


def test_cond_bias_rounds_like_rf_dit_prepare():
    assert R.cond_bias(2.0) == torch.tensor(0.69314718).to(torch.bfloat16).item()
    assert R.cond_bias(0.0) == float("-inf")


def _eager(q, k, v, B, S, heads, bias, scale, use_scale, causal):
    """transformers' eager attention in bf16 on the CPU -> (P [B, heads, S, S] bf16, out [B S, heads 64] bf16)"""
    P = torch.empty(B, heads, S, S, dtype=torch.bfloat16)
    out = torch.empty(B * S, heads * 64, dtype=torch.bfloat16)
    for b in range(B):
        r = slice(b * S, (b + 1) * S)
        qh, kh, vh = (t[r].view(S, heads, 64).transpose(0, 1) for t in (q, k, v))
        s = torch.matmul(qh, kh.transpose(1, 2))
        if use_scale:
            s = s * scale
        if bias is not None:
            s = s + bias
        if causal:
            s = s.masked_fill(torch.ones(S, S, dtype=torch.bool).triu(1), float("-inf"))
        P[b] = torch.softmax(s.float(), dim=-1).type_as(s)
        out[r] = torch.matmul(P[b], vh).transpose(0, 1).reshape(S, heads * 64)
    return P, out


def _text(name):
    B, S, heads, kind, off = R.TEXT_FIXTURES[name]
    qkv, bias = R.text_operands(B, S, heads, kind, off, R.seed_of(name))
    inner = heads * 64
    return (qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:], B, S, heads, bias) + R.text_args(kind)


@pytest.mark.parametrize("name", HOST_TEXT)
def test_text_reference_is_the_eager_sequence(name):
    """P bit for bit; with P V in float64 the outputs are equal bit for bit too.  torch's CPU bf16 matmul accumulates
    P V in fp32 in its own order, so a few outputs next to a rounding midpoint land an ulp away (outputs that cancel to
    far below their terms, a few ulps): within the text bars."""
    q, k, v, B, S, heads, bias, scale, use_scale, causal = args = _text(name)
    P, out = _eager(*args)
    for b in range(B):
        for h in range(heads):
            y = R.text_scores(q, k, b, h, S, bias, scale, use_scale, causal)
            assert torch.equal(R.bf(torch.softmax(y, dim=1)), P[b, h].float()), (b, h)
    ref, A = R.text_attention(*args)
    vh = v.view(B, S, heads, 64).transpose(1, 2).double()
    exact = (P.double() @ vh).float().to(torch.bfloat16).transpose(1, 2).reshape(B * S, heads * 64).float()
    assert torch.equal(ref, exact)
    same = (out.float() == ref).double().mean().item()
    print(f"[{name}] torch's bf16 matmul: identical {same:.5f}")
    assert R.text_passes(out.float(), ref, A)


@pytest.mark.parametrize("mut", R.TEXT_MUTATIONS)
def test_text_mutation_fails_the_bars(mut):
    caught = []
    for name in HOST_TEXT:
        args = _text(name)
        ref, A = R.text_attention(*args)
        if not R.text_passes(R.text_attention(*args, mut=(mut,))[0], ref, A):
            caught.append(name)
    print(f"{R.MUTATIONS[mut]}: fails the bars on {caught}")
    assert caught


def test_text_attention_hook_is_exported():
    from reflectionflow_b200 import _lib
    lib = R.declare(_lib.load())
    assert lib.rf_dbg_text_attention.restype is not None
