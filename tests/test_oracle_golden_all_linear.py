"""not-gpu: the all-linear oracle reproduces the golden vectors of tests/_all_linear_golden.py (outputs of the reference's
own code with a LoRA on every Linear) bit for bit, the targets outside train_flux/config.yaml:53 move the output far
beyond bf16 noise, and the factor generators keep the config.yaml:53 factors they drew before."""
import json
import os

import pytest
import torch

from oracle import cases as C
from oracle import flux_oracle as fo
from tests import _all_linear_golden as G

# full-width cases (D = 3072, K = 4096) are bit-exact only at the thread count they were minted with (the CPU bf16
# GEMM splits K by thread); like tests/test_oracle_golden.py, the bit-exact check covers the D = 256 cases
SMALL = [n for n, c in G.CASES.items() if c.heads == 2 and c.double * c.single <= 4]


@pytest.mark.parametrize("name", SMALL)
def test_oracle_matches_all_linear_golden_bit_exact(name):
    gold = G.load_golden()
    case = G.CASES[name]
    assert torch.equal(gold[name + "/rows"], C.golden_rows(name, case.n_img))
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // 2))
    out = G.run_oracle(case)
    assert torch.equal(C.golden_sample(gold, name, out), gold[name + "/bf16"]), \
        f"{name}: oracle drifted from the reference golden"


def test_all_linear_golden_error_budget_and_effect():
    meta = json.load(open(G.GOLDEN_FILE.replace(".safetensors", ".json")))["cases"]
    gold = G.load_golden()
    assert set(meta) == set(G.CASES)
    for name, case in G.CASES.items():
        assert torch.equal(gold[name + "/rows"], C.golden_rows(name, case.n_img))
        m = meta[name]
        assert 1e-3 < m["bf16_vs_fp32_mean"] < 3e-2, name
        # the new targets must matter far more than the bf16 error, or a dropped term would pass the parity bars
        assert m["all_linear_effect_mean"] > 20 * m["bf16_vs_fp32_mean"], name


def test_all_linear_factors_extend_the_config_targets():
    case = G.CASES["fwdB_al_small"]
    model, full = G.build_model(case)
    assert sorted(full) == G.all_linear_modules(model)
    gated, always = G.split(case.config(), full)
    ref = fo.make_lora_weights(model, case.config(), rank=case.lora_rank, seed=case.seed + 100)
    assert sorted(gated) == sorted(ref)
    assert all(torch.equal(gated[k][0], ref[k][0]) and torch.equal(gated[k][1], ref[k][1]) for k in ref)
    # context_embedder, 6 embedder Linears, norm_out.linear, proj_out; 8 per double block; none per single block
    assert len(always) == 9 + 8 * case.double


def test_synthetic_lora_all_linear_keeps_the_config_factors():
    from reflectionflow_b200.config import FluxDiTConfig
    from reflectionflow_b200.tts.reflectionflow import synthetic_lora
    cfg = FluxDiTConfig(num_layers=2, num_single_layers=1, num_attention_heads=2, joint_attention_dim=128,
                        pooled_projection_dim=64)
    base, full = synthetic_lora(cfg, rank=8), synthetic_lora(cfg, rank=8, targets="all-linear")
    for k, (a, b) in base.items():
        assert torch.equal(full[k][0], a) and torch.equal(full[k][1], b), k
    model = fo.FluxTransformer2DModel(fo.FluxConfig(num_layers=2, num_single_layers=1, num_attention_heads=2,
                                                    joint_attention_dim=128, pooled_projection_dim=64))
    mods = dict(model.named_modules())
    assert sorted(full) == G.all_linear_modules(model)
    for k, (a, b) in full.items():
        assert tuple(a.shape) == (8, mods[k].in_features) and tuple(b.shape) == (mods[k].out_features, 8), k
    with pytest.raises(ValueError):
        synthetic_lora(cfg, targets="attn-only")


def test_clear_lora_is_exported_and_checks_its_handle():
    from reflectionflow_b200 import _lib
    lib = _lib.load()
    assert hasattr(lib, "rf_dit_clear_lora")
    assert lib.rf_dit_clear_lora(None) != 0
