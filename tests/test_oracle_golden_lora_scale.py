"""not-gpu: the oracle reproduces the golden vectors of the scaled-LoRA cases (tests/_lora_scale_golden.py, outputs of
the reference's own code with lora_alpha != r and joint_attention_kwargs={"scale": s}) bit for bit, and the scaling
moves the output measurably."""
import json
import os

import pytest
import torch

from oracle import cases as C
from tests import _lora_scale_golden as G

# full-width cases (D = 3072, K = 4096) are bit-exact only at the thread count they were minted with (the CPU bf16
# GEMM splits K by thread); like tests/test_oracle_golden.py, the bit-exact check covers the D = 256 cases
SMALL = [n for n, c in G.CASES.items() if c.heads == 2]


@pytest.mark.parametrize("name", SMALL)
def test_oracle_matches_lora_scale_golden_bit_exact(name):
    gold = G.load_golden()
    case = G.CASES[name]
    assert torch.equal(gold[name + "/rows"], C.golden_rows(name, case.n_img))
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // 2))
    out = G.run_oracle(case)
    assert torch.equal(C.golden_sample(gold, name, out), gold[name + "/bf16"]), \
        f"{name}: oracle drifted from the reference golden"


def test_lora_scale_golden_error_budget_and_scale_effect():
    meta = json.load(open(G.GOLDEN_FILE.replace(".safetensors", ".json")))
    gold = G.load_golden()
    for name, case in G.CASES.items():
        assert torch.equal(gold[name + "/rows"], C.golden_rows(name, case.n_img))
        m = meta["cases"][name]
        assert 1e-3 < m["bf16_vs_fp32_mean"] < 2e-2
        assert m["effective_scaling"] == G.effective_scaling(case)
        if m["effective_scaling"] == 1.0:
            assert m["scale_effect_mean"] == 0.0
        else:
            # a scaling the reference applies moves its output; the cases with the adapter on the image rows move it
            # far beyond the bf16 error
            assert m["scale_effect_mean"] > 0.5 * m["bf16_vs_fp32_mean"]
            if case.model_config.get("latent_lora"):
                assert m["scale_effect_mean"] > 20 * m["bf16_vs_fp32_mean"]


def test_reference_scale_sequence_is_one_fp32_value():
    """peft's `scaling *= s` / `scaling /= s` around every call can drift in double; the fp32 value the bf16 term is
    multiplied by stays the same across the 28 calls of a loop for every case and for scales a user might pick."""
    for case in G.CASES.values():
        G.effective_scaling(case)
    base = G.CASES["denoiseB_28_s"]
    for alpha in (8, 16, 32, 64):
        for s in (0.0, 0.1, 0.3, 0.7, 0.75, 0.8, 0.9, 1.1, 1.3, 1.7, 2.5, -0.5):
            case = G.ScaleCase("probe", steps=28, lora_rank=32, lora_alpha=alpha, lora_scale=s)
            assert G.effective_scaling(case) == torch.tensor(alpha / 32 * s, dtype=torch.float32).item()
    assert base.alpha_over_r == 1.0
