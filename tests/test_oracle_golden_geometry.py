"""not-gpu: the oracle reproduces the golden vectors of the ragged-split masked-attention cases
(tests/_geometry_golden.py, outputs of the reference's own code) bit for bit."""
import json
import os

import pytest
import torch

from oracle import cases as C
from tests import _geometry_golden as G


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_matches_geometry_golden_bit_exact(name):
    gold = G.load_golden()
    case = G.CASES[name]
    assert (case.n_txt + case.n_img) % 128 != 0  # the split lies inside a 128-token tile
    assert torch.equal(gold[name + "/rows"], C.golden_rows(name, case.n_img))
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // 2))
    out = C.run_oracle(case)
    assert torch.equal(C.golden_sample(gold, name, out), gold[name + "/bf16"]), \
        f"{name}: oracle drifted from the reference golden"


def test_geometry_golden_error_budget():
    meta = json.load(open(G.GOLDEN_FILE.replace(".safetensors", ".json")))
    for name in G.CASES:
        assert 1e-3 < meta["cases"][name]["bf16_vs_fp32_mean"] < 2e-2
