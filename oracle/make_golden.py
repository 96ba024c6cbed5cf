"""Pin the oracle against the reference and mint tests/golden/.

Run in the BUILD CONTAINER only (needs /root/reference):  python -m oracle.make_golden

For every case of oracle/cases.py this
  1. runs the REFERENCE's own code — train_flux/flux/transformer.py::tranformer_forward (and
     generate.py::generate for the loop cases) with block.py / lora_controller.py underneath,
     imported unmodified from /root/reference over oracle/shims (restated diffusers leaf modules,
     peft-semantics LoRA layers) — on CPU in bf16;
  2. runs the oracle restatement (oracle/flux_oracle.py) on the same seeded inputs;
  3. requires the two to agree BIT FOR BIT;
  4. stores the output in tests/golden/flux_golden.safetensors (+ an fp32-arithmetic oracle
     output per case as the "true value" comparator for error-budget tests).
It also pins tts/utils.py::get_noises / prepare_latents_for_flux (seeded bf16 CPU noise)."""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import cases as C  # noqa: E402
from oracle import flux_oracle as fo  # noqa: E402
from oracle import ref_loader  # noqa: E402


def wrap_lora(model, lora, alpha_over_r=1.0):
    """Replace target Linears by peft-semantics LoRA layers (what pipe.load_lora_weights does)."""
    from peft.tuners.tuners_utils import LoraLinear
    for name, (A, B) in lora.items():
        parent_name, _, attr = name.rpartition(".")
        parent = model.get_submodule(parent_name) if parent_name else model
        base = getattr(parent, attr) if not attr.isdigit() else parent[int(attr)]
        wrapped = LoraLinear(base, A, B, alpha=alpha_over_r * A.shape[0])
        if attr.isdigit():
            parent[int(attr)] = wrapped
        else:
            setattr(parent, attr, wrapped)
    return model


class FakeCondition:
    """Stands in for train_flux/flux/condition.py::Condition with explicit latents (the real
    encode() samples the VAE posterior, SURVEY App. B.4)."""
    condition_type = "cot"

    def __init__(self, tokens, ids):
        self.tokens, self.ids = tokens, ids

    def encode(self, pipe, empty=False):
        return self.tokens, self.ids.clone(), torch.ones_like(self.ids[:, :1]) * 12


@torch.no_grad()
def run_reference(ns, case, dtype=torch.bfloat16):
    model, lora = C.build_model(case, dtype)
    if lora:
        wrap_lora(model, lora)
    x = C.build_inputs(case, dtype)
    mc = dict(case.model_config)
    if case.steps:
        from diffusers.pipelines import FluxPipeline
        pipe = FluxPipeline(model, dtype)
        conds = [FakeCondition(x["cond_latents"], x["cond_ids"])] if case.cond_size else None
        out = ns.generate.generate(pipe, conditions=conds, model_config=mc, default_lora=True,
                                   condition_scale=case.condition_scale,
                                   prompt_embeds=x["prompt_embeds"], pooled_prompt_embeds=x["pooled"],
                                   latents=x["latents"], height=case.height, width=case.width,
                                   num_inference_steps=case.steps, guidance_scale=case.guidance,
                                   output_type="latent", max_sequence_length=case.n_txt)
        return out.images
    if case.condition_scale != 1.0:  # generate.py:86-90
        for name, module in model.named_modules():
            if name.endswith(".attn"):
                module.c_factor = torch.ones(1, 1) * case.condition_scale
    return ns.transformer.tranformer_forward(
        model, condition_latents=x["cond_latents"], condition_ids=x["cond_ids"],
        condition_type_ids=None, model_config=mc, c_t=0, hidden_states=x["latents"],
        encoder_hidden_states=x["prompt_embeds"], pooled_projections=x["pooled"],
        timestep=x["timestep"], img_ids=x["img_ids"], txt_ids=x["txt_ids"], guidance=x["guidance"],
        joint_attention_kwargs=None, return_dict=False)[0]


def main():
    from safetensors.torch import save_file
    ns = ref_loader.load()
    torch.set_num_threads(os.cpu_count() or 1)
    out, meta = {}, {}
    for name, case in C.CASES.items():
        ref = run_reference(ns, case)
        ora = C.run_oracle(case)
        same = torch.equal(ref, ora)
        maxd = (ref.float() - ora.float()).abs().max().item()
        print(f"{name:22s} ref==oracle bit-exact: {same}  (max |d| = {maxd:g})  absmax={ref.float().abs().max():.3f}")
        if not same:
            raise SystemExit(f"oracle does not reproduce the reference on case {name}")
        out[name + "/bf16"] = ref.contiguous()
        # fp32-arithmetic oracle on the SAME bf16-valued weights/inputs: the "true value"
        m32, l32 = C.build_model(case, torch.bfloat16)
        m32 = m32.float()
        l32 = {k: (a.float(), b.float()) for k, (a, b) in l32.items()} if l32 else None
        x = C.build_inputs(case, torch.bfloat16)
        ls = fo.LoraSet(l32, 1.0) if l32 else None
        mc = C.oracle_model_config(case)
        f = lambda t: None if t is None else t.float()
        if case.steps:
            o32 = fo.denoise(m32, f(x["latents"]), f(x["prompt_embeds"]), f(x["pooled"]), case.steps,
                             case.guidance, f(x["img_ids"]), f(x["txt_ids"]), f(x["cond_latents"]),
                             f(x["cond_ids"]), mc, ls, scalar_dtype=torch.bfloat16)
        else:
            o32 = fo.transformer_forward(m32, f(x["latents"]), f(x["prompt_embeds"]), f(x["pooled"]),
                                         x["timestep"], f(x["img_ids"]), f(x["txt_ids"]),
                                         x["guidance"], f(x["cond_latents"]), f(x["cond_ids"]), mc, ls,
                                         scalar_dtype=torch.bfloat16)
        out[name + "/fp32"] = o32.contiguous()
        e = (ref.float() - o32).abs()
        meta[name] = {"bf16_vs_fp32_max": e.max().item(), "bf16_vs_fp32_mean": e.mean().item(),
                      "out_absmax": o32.abs().max().item()}
        print(f"{'':22s} reference(bf16) vs fp32 oracle: max {e.max():.4g} mean {e.mean():.4g}")

    # seeded noise: tts/utils.py:71-87,131-155
    u = ref_loader.load_tts_utils()
    for (h, w, seed) in [(256, 256, 1234), (1024, 1024, 42)]:
        ref = u.prepare_latents_for_flux(1, h, w, torch.manual_seed(seed), "cpu", torch.bfloat16)
        ora = fo.prepare_latents_for_flux(h, w, seed)
        assert torch.equal(ref, ora), "noise mismatch"
        out[f"noise/{h}x{w}@{seed}"] = ref[0, :8].contiguous()
        meta[f"noise/{h}x{w}@{seed}"] = {"sum": ref.float().sum().item()}
        print(f"noise {h}x{w}@{seed}: bit-exact, sum={ref.float().sum().item():.6f}")
    torch.manual_seed(0)
    ref_n = u.get_noises(2 ** 31 - 1, 3, 256, 256, device="cpu")
    torch.manual_seed(0)
    ora_n = fo.get_noises(2 ** 31 - 1, 3, 256, 256)
    assert list(ref_n) == list(ora_n) and all(torch.equal(ref_n[k], ora_n[k]) for k in ref_n)
    meta["get_noises/seed0"] = {"seeds": [int(k) for k in ref_n]}
    print("get_noises: seeds", list(ref_n))

    gdir = os.path.join(REPO, "tests", "golden")
    os.makedirs(gdir, exist_ok=True)
    for name in C.CASES:  # store a seeded sample of token rows per case (C.golden_rows); the stats above are full
        rows = C.golden_rows(name, out[name + "/bf16"].shape[1])
        out[name + "/rows"] = rows
        for kind in ("bf16", "fp32"):
            out[f"{name}/{kind}"] = out[f"{name}/{kind}"][:, rows].contiguous()
    save_file(out, os.path.join(gdir, "flux_golden.safetensors"))
    with open(os.path.join(gdir, "flux_golden.json"), "w") as fjson:
        json.dump({"generator": "oracle/make_golden.py", "reference_commit": "333d65a",
                   "torch": torch.__version__, "cases": meta}, fjson, indent=1)
    print("wrote", gdir)


if __name__ == "__main__":
    main()
