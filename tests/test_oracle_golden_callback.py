"""not-gpu: the oracle's callback loop reproduces the golden vectors of the callback cases (tests/_callback_golden.py,
outputs of the reference's own `generate(..., callback_on_step_end=...)`) bit for bit; every edit, T5 swap and
interrupt moves the output well beyond the bf16 error, and a no-op callback moves it not at all."""
import json
import os

import pytest
import torch

from oracle import cases as C
from tests import _callback_golden as G

# the cases run at D = 256 (heads 2): bit-exact at any thread count (see test_oracle_golden.py)
SMALL = [n for n, c in G.CASES.items() if c.heads == 2 and c.steps <= 4]


def _meta():
    return json.load(open(G.GOLDEN_FILE.replace(".safetensors", ".json")))["cases"]


@pytest.mark.parametrize("name", SMALL)
def test_oracle_matches_callback_golden_bit_exact(name):
    gold = G.load_golden()
    case = G.CASES[name]
    assert torch.equal(gold[name + "/rows"], C.golden_rows(name, case.n_img))
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // 2))
    out = G.run_oracle(case)
    assert torch.equal(C.golden_sample(gold, name, out), gold[name + "/bf16"]), \
        f"{name}: oracle drifted from the reference golden"


def test_callback_golden_error_budget_and_effects():
    meta, gold = _meta(), G.load_golden()
    assert set(meta) == set(G.CASES)
    for name, case in G.CASES.items():
        assert torch.equal(gold[name + "/rows"], C.golden_rows(name, case.n_img))
        m = meta[name]
        assert m["effective_scaling"] == G.effective_scaling(case)
        assert 1e-3 < m["bf16_vs_fp32_mean"] < 2e-2
        if case.kind == "noop":
            assert m["edit_effect_mean"] == 0.0, name
        else:
            # a dropped edit, swap or interrupt moves the output far beyond the bf16 error
            assert m["edit_effect_mean"] >= 5 * m["bf16_vs_fp32_mean"], name
