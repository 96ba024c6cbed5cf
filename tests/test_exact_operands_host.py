"""-m "not gpu": the exact-operand references of tests/_exact.py, on the CPU.

  * The operands really are exact: for every fixture, fp32 accumulation equals float64 accumulation, and the sum of
    the products' magnitudes stays below 2^(23 - e) (so any summation order is exact).
  * The bit-exact GPU tests (tests/test_gpu_gemm_groups.py) can fail: each reference with one rounding point moved
    or one scale misread (tests/_exact.py: MUTATIONS) differs from the correct reference on at least 1 % of the
    outputs of that fixture.
  * The ctypes mirror of rf_dbg_gemm_group has the library's layout."""
import pytest
import torch

from tests import _exact as E

# the LoRA fixtures: (M, K, N, sec_cols, pad, rank, scales); sec_cols > 0 is a stacked q|k|v launch
LORA_FIXTURES = {
    "qkv_pad64": (192, 256, 384, 128, 64, 48, (0.5, -0.75, 1 / 3)),
    "qkv_pad128": (160, 512, 768, 256, 128, 128, (2.0, 0.25, -1 / 3)),
    "single_k3072": (130, 3072, 256, 0, 64, 64, (1 / 3,)),
    "single_pad128": (128, 1024, 128, 0, 128, 96, (-0.75,)),
}


def lora_operands(M, K, N, sec_cols, pad, rank, seed=0):
    """x, W, bias and the zero-padded stacked factors A [nsec pad, K], B [N, pad] of one exact-operand LoRA group"""
    nsec = N // sec_cols if sec_cols else 1
    x, W = E.act((M, K), seed), E.weight((N, K), seed + 1)
    bias = E.randn((N,), seed + 2, 0.5)
    A = torch.zeros(nsec * pad, K, dtype=torch.bfloat16)
    B = torch.zeros(N, pad, dtype=torch.bfloat16)
    width = sec_cols or N
    for s in range(nsec):
        A[s * pad:s * pad + rank] = E.weight((rank, K), seed + 3 + s)
        B[s * width:(s + 1) * width, :rank] = E.lora_b((width, rank), seed + 6 + s)
    return x, W, bias, A, B


def lora_reference(fx, mut=()):
    M, K, N, sec_cols, pad, rank, scales = LORA_FIXTURES[fx]
    x, W, bias, A, B = lora_operands(M, K, N, sec_cols, pad, rank)
    exact = not mut
    T = E.lora_down(x, A, exact, mut)
    L = E.lora_up(T, B, scales, sec_cols, pad, exact, mut)
    return E.linear(x, W, bias, L=L, exact=exact, mut=mut)


def merge_operands(seed=0):
    W = E.act((256, 512), seed)
    A = E.dyadic((128, 512), 6, 64, seed + 1)
    B = E.weight((256, 128), seed + 2)
    return W, A, B


def _assert_fp32_accumulation_exact(a, w):
    E.gemm(a, w, exact=True)  # the magnitude bound
    assert torch.equal(a.float() @ w.float().t(), (a.double() @ w.double().t()).float())


@pytest.mark.parametrize("fx", list(LORA_FIXTURES))
def test_lora_fixture_operands_are_exact(fx):
    M, K, N, sec_cols, pad, rank, scales = LORA_FIXTURES[fx]
    x, W, bias, A, B = lora_operands(M, K, N, sec_cols, pad, rank)
    _assert_fp32_accumulation_exact(x, W)
    _assert_fp32_accumulation_exact(x, A)
    T = E.lora_down(x, A)
    width = sec_cols or N
    for s in range(N // width):
        _assert_fp32_accumulation_exact(T[:, s * pad:(s + 1) * pad], B[s * width:(s + 1) * width])
    # the values need more than bf16's 8 significant bits: rounding points move bits
    assert (E.gemm(x, W) != E.linear(x, W)).float().mean() > 0.25
    assert (E.gemm(x, A) != T).float().mean() > 0.1  # (the rank padding is zero)


def test_merge_fixture_operands_are_exact():
    W, A, B = merge_operands()
    _assert_fp32_accumulation_exact(B, A.t())
    d = E.gemm(B, A.t())
    assert (d != E.bf(d)).float().mean() > 0.25


def _lora_mutations(fx):
    sec_cols, scales = LORA_FIXTURES[fx][3], LORA_FIXTURES[fx][6]
    muts = ["L_unrounded", "T_unrounded", "lora_before_bias"]
    if sec_cols and len(set(scales)) > 1:
        muts.append("scale_sec0")
    return [(fx, m) for m in muts]


@pytest.mark.parametrize("fx,mut", [c for fx in LORA_FIXTURES for c in _lora_mutations(fx)])
def test_lora_mutation_changes_the_reference(fx, mut):
    good, bad = lora_reference(fx), lora_reference(fx, (mut,))
    frac = (good != bad).float().mean().item()
    print(f"[{fx}] {E.MUTATIONS[mut]}: {frac:.3f} of outputs differ")
    assert frac >= 0.01


def test_merge_mutation_changes_the_reference():
    W, A, B = merge_operands()
    for s in (1 / 3, -0.75):
        good, bad = E.lora_merge(W, A, B, s), E.lora_merge(W, A, B, s, exact=False, mut=("merge_thrice",))
        frac = (good != bad).float().mean().item()
        print(f"[merge s={s:.4g}] {E.MUTATIONS['merge_thrice']}: {frac:.3f} of outputs differ")
        assert frac >= 0.01


def test_section_scales_one_equals_the_unscaled_term():
    """s = 1 is the identity on bf16(L): the reference of a unit scale is the unscaled peft term"""
    M, K, N, sec_cols, pad, rank, _ = LORA_FIXTURES["qkv_pad64"]
    x, W, bias, A, B = lora_operands(M, K, N, sec_cols, pad, rank)
    T = E.lora_down(x, A)
    L1 = E.lora_up(T, B, (1.0, 1.0, 1.0), sec_cols, pad)
    plain = torch.cat([E.bf(E.gemm(T[:, s * pad:(s + 1) * pad], B[s * sec_cols:(s + 1) * sec_cols]))
                       for s in range(3)], 1)
    assert torch.equal(L1, plain)


def test_gemm_group_mirror_matches_the_library_layout():
    import ctypes
    from reflectionflow_b200 import _lib
    lib = E.declare(_lib.load())
    assert lib.rf_dbg_gemm_group_size() == ctypes.sizeof(E.GemmGroup)
