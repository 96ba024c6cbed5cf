"""not-gpu: the oracle's guided loop reproduces the golden vectors of the image-guidance cases
(tests/_image_guidance_golden.py, outputs of the reference's own `generate(..., image_guidance_scale=s)`) bit for bit;
guidance and the uncond latents move the output well beyond the bf16 error; the guidance scalar rounds as fp32."""
import json
import os

import pytest
import torch

from oracle import cases as C
from tests import _image_guidance_golden as G

# full-width cases are bit-exact only at the thread count they were minted with (see test_oracle_golden.py)
SMALL = [n for n, c in G.CASES.items() if c.heads == 2]


def _meta():
    return json.load(open(G.GOLDEN_FILE.replace(".safetensors", ".json")))["cases"]


@pytest.mark.parametrize("name", SMALL)
def test_oracle_matches_image_guidance_golden_bit_exact(name):
    gold = G.load_golden()
    case = G.CASES[name]
    assert torch.equal(gold[name + "/rows"], C.golden_rows(name, case.n_img))
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // 2))
    out = G.run_oracle(case)
    assert torch.equal(C.golden_sample(gold, name, out), gold[name + "/bf16"]), \
        f"{name}: oracle drifted from the reference golden"


def test_image_guidance_golden_error_budget_and_effects():
    meta, gold = _meta(), G.load_golden()
    assert set(meta) == set(G.CASES)
    for name, case in G.CASES.items():
        assert torch.equal(gold[name + "/rows"], C.golden_rows(name, case.n_img))
        m = meta[name]
        assert m["image_guidance_scale"] == case.image_guidance_scale
        assert m["effective_scaling"] == G.effective_scaling(case)
        assert 1e-3 < m["bf16_vs_fp32_mean"] < 2e-2
        # a dropped uncond branch moves the output far beyond the bf16 error
        assert m["guidance_effect_mean"] > 5 * m["bf16_vs_fp32_mean"], name
        assert ("uncond_effect_mean" in m) == case.distinct_uncond
        if not case.distinct_uncond:
            continue
        if not case.model_config.get("union_cond_attn", True):
            # the image rows do not attend to the condition rows: U_i cannot reach the output
            assert m["uncond_effect_mean"] == 0.0, name
        else:
            # U_i = C0 instead of the step's own slice moves it beyond the bf16 error; the uncond branch enters
            # v = c + (1 - s) (u - c) scaled by 1 - s, so s = 1.3 moves it least
            bar = 1.5 if abs(1 - case.image_guidance_scale) >= 0.5 else 1.2
            assert m["uncond_effect_mean"] > bar * m["bf16_vs_fp32_mean"], name


def test_guidance_scalar_rounds_as_fp32():
    """`unc_pred + s * (noise_pred - unc_pred)` on bf16 tensors with a Python float s is
    bf16(u + bf16(fp32(s) * bf16(c - u))); a double or a bf16 scalar rounds differently at s = 1.3."""
    g = torch.Generator().manual_seed(0)
    c, u = (torch.randn(65536, generator=g).to(torch.bfloat16) for _ in range(2))
    s = 1.3
    torch_v = u + s * (c - u)
    d = (c - u).float()

    def combine(prod):
        return (u.float() + prod.to(torch.bfloat16).float()).to(torch.bfloat16)

    assert torch.equal(torch_v, combine(torch.tensor(s, dtype=torch.float32) * d))
    assert not torch.equal(torch_v, combine(s * d.double()))
    assert not torch.equal(torch_v, combine(torch.tensor(s).to(torch.bfloat16).float() * d))


def test_lora_call_scale_is_one_fp32_value_over_two_calls_per_step():
    for case in G.CASES.values():
        G.effective_scaling(case)
    assert G.effective_scaling(G.CASES["ig_lora07"]) == torch.tensor(0.7, dtype=torch.float32).item()
