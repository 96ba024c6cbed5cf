"""CPU checks of tests/_text_ref.py, the references the text-encoder kernel tests (test_gpu_text_ops.py) compare against:

  * each restatement equals transformers' own module run by torch in bf16 on the CPU: T5LayerNorm on the row-norm
    fixtures, NewGELUActivation and QuickGELUActivation on every finite bf16 value, the gated product on the random
    pairs, CLIPTextEmbeddings.  The affine LayerNorm is nn.LayerNorm(eps=1e-5) evaluated in float64 and rounded once:
    torch's bf16 LayerNorm on the CPU computes x rstd - mean rstd in fp32 and loses bits to that cancellation (1-2 % of
    the outputs at mean / std = 128), so its CPU bits are not a reference; the GPU test compares with F.layer_norm on
    the device;
  * every entry of MUTATIONS changes at least 1 % of the outputs of a fixture the GPU file runs, except `cube_once`,
    which moves 7 of the 65280 finite bf16 values through gelu_new: the GPU test compares all of them bit for bit;
  * the ctypes declarations match the hooks' C signatures."""
import os
import re

import pytest
import torch

from tests import _exact as E
from tests import _text_ref as R

BF = torch.bfloat16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _changed(a, b):
    return int((a.to(BF).view(torch.int16) != b.to(BF).view(torch.int16)).sum())


# ------------------------------------------------------------------------------------ restatements = transformers
@pytest.mark.parametrize("dim", R.NORM_DIMS)
def test_t5_layernorm_is_transformers(dim):
    from transformers.models.t5.modeling_t5 import T5LayerNorm
    for rows in R.NORM_ROWS:
        for case in R.NORM_CASES[0]:
            x, w, _ = R.norm_inputs(rows, dim, case, 0)
            m = T5LayerNorm(dim, eps=R.T5_EPS).to(BF)
            with torch.no_grad():
                m.weight.copy_(w)
                want = m(x)
            assert _changed(R.t5_layernorm(x, w), want) == 0, (rows, case)


@pytest.mark.parametrize("dim", R.NORM_DIMS)
def test_layer_norm_is_nn_layernorm(dim):
    for rows in R.NORM_ROWS:
        for case in R.NORM_CASES[1]:
            x, w, b = R.norm_inputs(rows, dim, case, 1)
            m = torch.nn.LayerNorm(dim, eps=R.CLIP_EPS).double()
            with torch.no_grad():
                m.weight.copy_(w.double())
                m.bias.copy_(b.double())
                want = E.bf(m(x.double()).float())
            assert _changed(R.layer_norm(x, w, b), want) == 0, (rows, case)


def test_gelu_new_is_transformers_on_every_bf16_value():
    from transformers.activations import NewGELUActivation
    v = R.all_finite_bf16()
    assert v.numel() == 65280
    assert _changed(R.gelu_new(v), NewGELUActivation()(v)) == 0


def test_quick_gelu_is_transformers_on_every_bf16_value():
    from transformers.activations import QuickGELUActivation
    v = R.all_finite_bf16()
    assert _changed(R.quick_gelu(v), QuickGELUActivation()(v)) == 0


def test_gated_product_is_t5_dense_gated_act_dense():
    """T5DenseGatedActDense (gated-gelu, bf16) on rows [a, b] with projections that pick a (wi_0) and b (wi_1): exact
    selections, so what reaches wo is the module's hidden_gelu * hidden_linear of (a, b), signed zeros included"""
    from transformers import T5Config
    from transformers.models.t5.modeling_t5 import T5DenseGatedActDense
    a, b = R.random_pairs()
    m = T5DenseGatedActDense(T5Config(d_model=2, d_ff=1, feed_forward_proj="gated-gelu", dropout_rate=0.0)).eval()
    assert m.act.__class__.__name__ == "NewGELUActivation"
    m = m.to(BF)
    seen = []
    m.wo.register_forward_hook(lambda mod, inp, out: seen.append(inp[0]))
    with torch.no_grad():
        m.wi_0.weight.copy_(torch.tensor([[1.0, 0.0]]))
        m.wi_1.weight.copy_(torch.tensor([[0.0, 1.0]]))
        m(torch.stack([a, b], -1))
    assert _changed(R.gated(a, b), seen[0][:, 0].contiguous()) == 0


@pytest.mark.parametrize("S", [20, 77])
def test_embed_is_clip_text_embeddings(S):
    from transformers import CLIPTextConfig
    from transformers.models.clip.modeling_clip import CLIPTextEmbeddings
    m = CLIPTextEmbeddings(CLIPTextConfig(vocab_size=1000, hidden_size=256, max_position_embeddings=77)).to(BF)
    g = torch.Generator().manual_seed(S)
    ids = torch.randint(0, 1000, (3, S), generator=g)
    with torch.no_grad():
        want = m(input_ids=ids).reshape(3 * S, 256)
    got = R.embed(ids.flatten(), m.token_embedding.weight.detach(), m.position_embedding.weight.detach(), S)
    assert _changed(got, want) == 0
    assert torch.equal(R.embed(ids.flatten(), m.token_embedding.weight.detach()), m.token_embedding(ids).reshape(
        3 * S, 256).float())


# ------------------------------------------------------------------------------------ mutations
def _mutated(mut):
    """(reference, mutated reference) on a fixture test_gpu_text_ops.py runs"""
    if mut == "gelu_fused":
        a, b = R.random_pairs()
        return R.gated(a, b), R.gated(a, b, (mut,))
    if mut == "cube_once":
        v = R.all_finite_bf16()
        return R.gelu_new(v), R.gelu_new(v, (mut,))
    if mut == "rms_unrounded":
        x, w, _ = R.norm_inputs(77, 1024, "unit", 0)
        return R.t5_layernorm(x, w), R.t5_layernorm(x, w, mut=(mut,))
    if mut == "ln_eps":
        x, w, b = R.norm_inputs(77, 768, "small", 1)
        return R.layer_norm(x, w, b), R.layer_norm(x, w, b, mut=(mut,))
    if mut == "ln_no_mean":
        x, w, b = R.norm_inputs(77, 768, "unit", 1)
        return R.layer_norm(x, w, b), R.layer_norm(x, w, b, mut=(mut,))
    if mut == "quick_unrounded":
        v = R.all_finite_bf16()
        return R.quick_gelu(v), R.quick_gelu(v, (mut,))
    if mut == "pos_row_t":
        g = torch.Generator().manual_seed(20)
        table, pos = torch.randn(1000, 768, generator=g).to(BF), torch.randn(77, 768, generator=g).to(BF)
        ids = torch.randint(0, 1000, (3 * 20,), generator=g)
        return R.embed(ids, table, pos, 20), R.embed(ids, table, pos, 20, mut=(mut,))
    if mut == "gather_batch0":
        x = E.randn((3 * 77, 768), 77 + 768)
        pos = torch.tensor([0, 76, 38], dtype=torch.int32)
        return R.gather(x, pos, 77), R.gather(x, pos, 77, mut=(mut,))
    raise KeyError(mut)


@pytest.mark.parametrize("mut", sorted(R.MUTATIONS))
def test_mutation_is_caught(mut):
    ref, bad = _mutated(mut)
    n = _changed(ref, bad)
    print(f"{mut}: {n} of {ref.numel()} ({n / ref.numel():.4f}) outputs change")
    if mut == "cube_once":
        # bit-exact over every finite bf16 value on the GPU: the 7 moved values (-2.734375, -2.453125, -2.125,
        # -0.90625, -0.828125, 0.90625, 2.734375) are among them
        assert n == 7
    else:
        assert n >= 0.01 * ref.numel()


# ------------------------------------------------------------------------------------ the binding
def test_hook_declarations_match_the_c_signatures():
    src = open(os.path.join(ROOT, "reflectionflow_b200", "csrc", "rf_api.cu")).read()
    kinds = {"int": "ci", "int64_t": "cl", "float": "cf"}
    for name, args in R.HOOKS.items():
        m = re.search(r"\bint " + name + r"\(([^)]*)\)", src)
        assert m, f"{name} is not defined in rf_api.cu"
        params = [p.strip() for p in m.group(1).replace("\n", " ").split(",") if p.strip() and p.strip() != "void"]
        got = ["vp" if "*" in p else kinds[p.rsplit(" ", 1)[0].strip()] for p in params]
        assert got == args.split(), (name, got, args)
    header = open(os.path.join(ROOT, "include", "rf_b200.h")).read()
    assert "rf_dbg_text" not in header and "rf_dbg_t5" not in header  # test hooks stay out of the public ABI
