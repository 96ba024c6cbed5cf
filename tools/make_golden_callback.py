#!/usr/bin/env python
"""Mint tests/golden/flux_golden_callback.safetensors (+ .json) for the cases of tests/_callback_golden.py.

Needs the original project's tree (RF_REFERENCE_ROOT, default /root/reference).  For every case it runs the
reference's own `generate(..., callback_on_step_end=cb, callback_on_step_end_tensor_inputs=...)` on CPU in bf16 with
the case's scripted callback (an image-guided case also with the scripted condition of
tools/make_golden_image_guidance.py), requires the oracle's loop to agree bit for bit, and stores a seeded sample of
token rows of the bf16 output and of the fp32-arithmetic oracle output.  `edit_effect_mean` in the json, the distance
from the same case without a callback, keeps a dropped edit, swap or interrupt from hiding under the bf16 error.
The tool also asserts that the callback saw exactly the steps the case executes, with t = scheduler.timesteps[i]."""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

from oracle import cases as C  # noqa: E402
from oracle import flux_oracle as fo  # noqa: E402
from oracle import ref_loader  # noqa: E402
from oracle.make_golden import wrap_lora  # noqa: E402
from tests import _callback_golden as G  # noqa: E402
import make_golden_image_guidance as IGT  # noqa: E402
import make_golden_lora_scale as LST  # noqa: E402


@torch.no_grad()
def run_reference(ns, case, dtype=torch.bfloat16):
    LoraLinear = LST._peft_layers(ns)
    model, lora = C.build_model(case, dtype)
    if lora:
        wrap_lora(model, lora)
        for m in model.modules():
            if isinstance(m, LoraLinear):
                r = m.lora_A["default"].weight.shape[0]
                m.r = {"default": r}
                m.lora_alpha = {"default": r}
    x = C.build_inputs(case, dtype)
    from diffusers.pipelines import FluxPipeline
    pipe = FluxPipeline(model, dtype)
    conditions = None
    if case.cond_size:
        U = G.uncond_latents(case, dtype) if case.image_guidance_scale != 1.0 else []
        conditions = [IGT.ScriptedCondition(x["cond_latents"], U, x["cond_ids"])]
    cb, seen = G.scripted_callback(case), []

    def recording_cb(p, i, t, kw):
        assert set(kw) == set(case.tensor_inputs)
        seen.append((i, t.item()))
        return cb(p, i, t, kw)
    jak = {"scale": case.lora_scale} if case.lora_scale != 1.0 else None
    out = ns.generate.generate(pipe, conditions=conditions, model_config=dict(case.model_config), default_lora=True,
                               condition_scale=case.condition_scale, image_guidance_scale=case.image_guidance_scale,
                               joint_attention_kwargs=jak, prompt_embeds=x["prompt_embeds"],
                               pooled_prompt_embeds=x["pooled"], latents=x["latents"], height=case.height,
                               width=case.width, num_inference_steps=case.steps, guidance_scale=case.guidance,
                               output_type="latent", max_sequence_length=case.n_txt,
                               callback_on_step_end=recording_cb,
                               callback_on_step_end_tensor_inputs=list(case.tensor_inputs)).images
    ts, _ = fo.flow_match_sigmas(case.steps, case.n_img)
    n_run = case.edit_step + 1 if case.kind.endswith("interrupt") else case.steps
    assert seen == [(i, ts[i].item()) for i in range(n_run)], seen
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
        m = {"effective_scaling": G.effective_scaling(case),
             "edit_effect_mean": (ora.float() - G.run_oracle(case, with_callback=False).float()).abs().mean().item()}
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
        json.dump({"generator": "tools/make_golden_callback.py", "torch": torch.__version__, "cases": meta},
                  fjson, indent=1)
    print("wrote", G.GOLDEN_FILE)


if __name__ == "__main__":
    main()
