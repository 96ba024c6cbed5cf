#!/usr/bin/env python
"""Mint tests/golden/flux_golden_image_guidance.safetensors (+ .json) for the cases of tests/_image_guidance_golden.py.

Needs the original project's tree (RF_REFERENCE_ROOT, default /root/reference).  For every case it runs the
reference's own `generate(..., image_guidance_scale=s)` on CPU in bf16 with a scripted condition: its first `encode`
returns C0, and each later `encode(empty=True)` returns the next U_i (the tool asserts `empty=True` was passed and
that every U_i was used).  It requires the oracle to agree bit for bit and stores a seeded sample of token rows of
the bf16 output and of the fp32-arithmetic oracle output.  Two numbers in the json keep a dropped branch or a wrong
U slice from hiding under the bf16 error: `guidance_effect_mean`, the distance from the same case at s = 1, and
for cases with distinct U_i `uncond_effect_mean`, the distance from U_i = C0.

A case with a LoRA call scale uses the peft scale / unscale patches of tools/make_golden_lora_scale.py: the
reference scales its layers around each of the two transformer calls per step."""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

from oracle import cases as C  # noqa: E402
from oracle import ref_loader  # noqa: E402
from oracle.make_golden import wrap_lora  # noqa: E402
from tests import _image_guidance_golden as G  # noqa: E402
import make_golden_lora_scale as LST  # noqa: E402


class ScriptedCondition:
    """train_flux/flux/condition.py::Condition as the guided loop sees it: C0 from the first `encode`, then U_i
    from the i-th `encode(empty=True)` (generate.py:251)."""
    condition_type = "cot"

    def __init__(self, c0, uncond, ids):
        self.c0, self.uncond, self.ids = c0, list(uncond), ids
        self.n_encodes = 0

    def encode(self, pipe, empty=False):
        assert empty == (self.n_encodes > 0), "the first encode is the condition, every later one is empty=True"
        tokens = self.c0 if self.n_encodes == 0 else self.uncond[self.n_encodes - 1]
        self.n_encodes += 1
        return tokens, self.ids.clone(), torch.ones_like(self.ids[:, :1]) * 12


@torch.no_grad()
def run_reference(ns, case, dtype=torch.bfloat16):
    LoraLinear = LST._peft_layers(ns)
    model, lora = C.build_model(case, dtype)
    wrap_lora(model, lora)
    for m in model.modules():
        if isinstance(m, LoraLinear):
            r = m.lora_A["default"].weight.shape[0]
            m.r = {"default": r}
            m.lora_alpha = {"default": r}
    x = C.build_inputs(case, dtype)
    from diffusers.pipelines import FluxPipeline
    pipe = FluxPipeline(model, dtype)
    cond = ScriptedCondition(x["cond_latents"], G.uncond_latents(case, dtype), x["cond_ids"])
    jak = {"scale": case.lora_scale} if case.lora_scale != 1.0 else None
    out = ns.generate.generate(pipe, conditions=[cond], model_config=dict(case.model_config), default_lora=True,
                               condition_scale=case.condition_scale, image_guidance_scale=case.image_guidance_scale,
                               joint_attention_kwargs=jak, prompt_embeds=x["prompt_embeds"],
                               pooled_prompt_embeds=x["pooled"], latents=x["latents"], height=case.height,
                               width=case.width, num_inference_steps=case.steps, guidance_scale=case.guidance,
                               output_type="latent", max_sequence_length=case.n_txt).images
    assert cond.n_encodes == case.steps + 1, cond.n_encodes
    # 2 calls per step: the layers end where the scale / unscale sequence says the next call would start
    s = case.lora_scale
    last = LST.G.reference_scalings(LST.G.ScaleCase("probe", steps=2 * case.steps, lora_rank=32, lora_scale=s))[-1]
    after = 1.0 if s == 0 else (last / s if s != 1 else last)
    for m in model.modules():
        if isinstance(m, LoraLinear):
            assert m.scaling["default"] == after, (m.scaling, after)
    return out


def main():
    from safetensors.torch import save_file
    ns = ref_loader.load()
    torch.set_num_threads(os.cpu_count() or 1)
    only = set(sys.argv[1:])
    out, meta = {}, {}
    for name, case in G.CASES.items():
        if only and name not in only:
            continue
        ref = run_reference(ns, case)
        ora = G.run_oracle(case)
        same = torch.equal(ref, ora)
        guidance_effect = (ora.float() - G.run_oracle(case, s=1.0).float()).abs().mean().item()
        m = {"image_guidance_scale": case.image_guidance_scale, "effective_scaling": G.effective_scaling(case),
             "guidance_effect_mean": guidance_effect}
        if case.distinct_uncond:
            m["uncond_effect_mean"] = (ora.float() - G.run_oracle(case, distinct=False).float()).abs().mean().item()
        print(f"{name:12s} ref==oracle bit-exact: {same}  {m}", flush=True)
        if not same:
            raise SystemExit(f"oracle does not reproduce the reference on case {name}")
        o32 = G.fp32_oracle(case)
        e = (ref.float() - o32).abs()
        meta[name] = dict(m, bf16_vs_fp32_max=e.max().item(), bf16_vs_fp32_mean=e.mean().item(),
                          out_absmax=o32.abs().max().item())
        print(f"{'':12s} reference(bf16) vs fp32 oracle: max {e.max():.4g} mean {e.mean():.4g}", flush=True)
        rows = C.golden_rows(name, ref.shape[1])
        out[name + "/rows"] = rows
        out[name + "/bf16"] = ref[:, rows].contiguous()
        out[name + "/fp32"] = o32[:, rows].contiguous()
    if only:
        print("subset run: nothing written")
        return
    save_file(out, G.GOLDEN_FILE)
    with open(G.GOLDEN_FILE.replace(".safetensors", ".json"), "w") as fjson:
        json.dump({"generator": "tools/make_golden_image_guidance.py", "torch": torch.__version__, "cases": meta},
                  fjson, indent=1)
    print("wrote", G.GOLDEN_FILE)


if __name__ == "__main__":
    main()
