#!/usr/bin/env python
"""Mint tests/golden/flux_golden_lora_scale.safetensors (+ .json) for the cases of tests/_lora_scale_golden.py.

Needs the original project's tree (RF_REFERENCE_ROOT, default /root/reference).  For every case it runs the
reference's own `tranformer_forward` / `generate` on CPU in bf16, with peft-semantics LoRA layers whose scaling is
lora_alpha / r and with `joint_attention_kwargs={"scale": s}`, requires the oracle to agree bit for bit, and stores a
seeded sample of token rows of the bf16 output and of the fp32-arithmetic oracle output.  It also records how far
the scaling moves the output (the same case at scaling 1), so a scale that is silently dropped cannot hide under the
bf16 error budget.

The reference scales and unscales its LoRA layers around every transformer call (`scale_lora_layers` /
`unscale_lora_layers`).  The peft LoRA layer of oracle/shims only has `scale_layer`, so this tool gives it peft's
`unscale_layer` and `set_scale`, and gives the reference diffusers' `unscale_lora_layers`, for the run."""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import cases as C  # noqa: E402
from oracle import ref_loader  # noqa: E402
from oracle.make_golden import FakeCondition, wrap_lora  # noqa: E402
from tests import _lora_scale_golden as G  # noqa: E402


def _unscale_layer(self, scale=None):
    """peft LoraLayer.unscale_layer"""
    for a in self.active_adapters:
        if a not in self.scaling:
            continue
        if scale is None:
            self.scaling[a] = self.lora_alpha[a] / self.r[a]
        else:
            self.scaling[a] /= scale


def _set_scale(self, adapter, scale):
    """peft LoraLayer.set_scale"""
    if adapter in self.scaling:
        self.scaling[adapter] = scale * self.lora_alpha[adapter] / self.r[adapter]


def _unscale_lora_layers(model, weight=None):
    """diffusers.utils.peft_utils.unscale_lora_layers"""
    if weight is None or weight == 1.0:
        return
    for m in model.modules():
        if hasattr(m, "unscale_layer") and hasattr(m, "lora_A"):
            if weight != 0:
                m.unscale_layer(weight)
            else:
                for a in m.active_adapters:
                    m.set_scale(a, 1.0)


def _peft_layers(ns):
    from peft.tuners.tuners_utils import LoraLinear
    LoraLinear.unscale_layer = _unscale_layer
    LoraLinear.set_scale = _set_scale
    ns.transformer.unscale_lora_layers = _unscale_lora_layers
    return LoraLinear


@torch.no_grad()
def run_reference(ns, case, dtype=torch.bfloat16):
    LoraLinear = _peft_layers(ns)
    model, lora = C.build_model(case, dtype)
    wrap_lora(model, lora, alpha_over_r=case.alpha_over_r)
    for m in model.modules():
        if isinstance(m, LoraLinear):
            r = m.lora_A["default"].weight.shape[0]
            m.r = {"default": r}
            m.lora_alpha = {"default": case.alpha_over_r * r}
    x = C.build_inputs(case, dtype)
    mc = dict(case.model_config)
    jak = {"scale": case.lora_scale}
    if case.steps:
        from diffusers.pipelines import FluxPipeline
        pipe = FluxPipeline(model, dtype)
        conds = [FakeCondition(x["cond_latents"], x["cond_ids"])] if case.cond_size else None
        out = ns.generate.generate(pipe, conditions=conds, model_config=mc, default_lora=True,
                                   condition_scale=case.condition_scale, joint_attention_kwargs=jak,
                                   prompt_embeds=x["prompt_embeds"], pooled_prompt_embeds=x["pooled"],
                                   latents=x["latents"], height=case.height, width=case.width,
                                   num_inference_steps=case.steps, guidance_scale=case.guidance,
                                   output_type="latent", max_sequence_length=case.n_txt)
        out = out.images
    else:
        out = ns.transformer.tranformer_forward(
            model, condition_latents=x["cond_latents"], condition_ids=x["cond_ids"], condition_type_ids=None,
            model_config=mc, c_t=0, hidden_states=x["latents"], encoder_hidden_states=x["prompt_embeds"],
            pooled_projections=x["pooled"], timestep=x["timestep"], img_ids=x["img_ids"], txt_ids=x["txt_ids"],
            guidance=x["guidance"], joint_attention_kwargs=jak, return_dict=False)[0]
    # the layers end where G.reference_scalings says the next call would start
    s, last = case.lora_scale, G.reference_scalings(case)[-1]
    after = case.alpha_over_r if s == 0 else (last / s if s != 1 else last)
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
        s32 = G.effective_scaling(case)
        ref = run_reference(ns, case)
        ora = G.run_oracle(case)
        same = torch.equal(ref, ora)
        unit = G.run_oracle(case, scaling=1.0)
        effect = (ora.float() - unit.float()).abs().mean().item()
        print(f"{name:20s} s32 {s32!r} ref==oracle bit-exact: {same}  (scale effect: mean |d| {effect:.4g})",
              flush=True)
        if not same:
            raise SystemExit(f"oracle does not reproduce the reference on case {name}")
        o32 = G.fp32_oracle(case)
        e = (ref.float() - o32).abs()
        meta[name] = {"bf16_vs_fp32_max": e.max().item(), "bf16_vs_fp32_mean": e.mean().item(),
                      "out_absmax": o32.abs().max().item(), "effective_scaling": s32, "scale_effect_mean": effect}
        rows = C.golden_rows(name, ref.shape[1])
        out[name + "/rows"] = rows
        out[name + "/bf16"] = ref[:, rows].contiguous()
        out[name + "/fp32"] = o32[:, rows].contiguous()
    if only:
        print("subset run: nothing written")
        return
    save_file(out, G.GOLDEN_FILE)
    with open(G.GOLDEN_FILE.replace(".safetensors", ".json"), "w") as fjson:
        json.dump({"generator": "tools/make_golden_lora_scale.py", "torch": torch.__version__, "cases": meta},
                  fjson, indent=1)
    print("wrote", G.GOLDEN_FILE)


if __name__ == "__main__":
    main()
