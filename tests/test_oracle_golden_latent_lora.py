"""not-gpu: the oracle reproduces the golden vectors of the `latent_lora: True` cases (tests/_latent_lora_golden.py,
outputs of the reference's own code) bit for bit, and the flag moves the output far beyond the bf16 error budget."""
import json
import os

import pytest
import torch

from oracle import cases as C
from tests import _latent_lora_golden as G


# full-width cases (D = 3072, K = 4096) are bit-exact only at the thread count they were minted with (the CPU bf16
# GEMM splits K by thread); like tests/test_oracle_golden.py, the bit-exact check covers the D = 256 cases
SMALL = [n for n, c in G.CASES.items() if c.heads == 2]


@pytest.mark.parametrize("name", SMALL)
def test_oracle_matches_latent_lora_golden_bit_exact(name):
    gold = G.load_golden()
    case = G.CASES[name]
    assert case.model_config.get("latent_lora") is True
    assert torch.equal(gold[name + "/rows"], C.golden_rows(name, case.n_img))
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // 2))
    out = C.run_oracle(case)
    assert torch.equal(C.golden_sample(gold, name, out), gold[name + "/bf16"]), \
        f"{name}: oracle drifted from the reference golden"


def test_latent_lora_golden_error_budget_and_effect():
    meta = json.load(open(G.GOLDEN_FILE.replace(".safetensors", ".json")))
    for name in G.CASES:
        assert torch.equal(G.load_golden()[name + "/rows"], C.golden_rows(name, G.CASES[name].n_img))
        m = meta["cases"][name]
        assert 1e-3 < m["bf16_vs_fp32_mean"] < 2e-2
        # a missing LoRA term on the image / text rows could not hide under the bf16 error
        assert m["latent_lora_effect_mean"] > 20 * m["bf16_vs_fp32_mean"]
