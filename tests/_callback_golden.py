"""DiT golden cases with per-step callbacks (`callback_on_step_end`, `pipe._interrupt`; generate.py:217-290).  Minted
by tools/make_golden_callback.py with the reference's own `generate()` into tests/golden/flux_golden_callback.safetensors.

The reference's loop, per step i:
  if pipe.interrupt: continue
  latents = scheduler.step(forward(latents, prompt_embeds, t_i), t_i, latents)   (image-guided: two forwards)
  out = callback_on_step_end(pipe, i, t_i, {k: locals()[k] for k in tensor_inputs})
  latents = out.pop("latents", latents); prompt_embeds = out.pop("prompt_embeds", prompt_embeds)

`scripted_callback` is the case's callback: a no-op, a seeded latents edit, a seeded T5-state swap, an interrupt, or a
latents edit with an interrupt, at `edit_step`.  It is a pure function of (case, i, tensors), so the reference, the oracle and the CUDA path run the
same one."""
import os
from dataclasses import dataclass, field
from typing import List, Optional

import torch

from oracle import cases as C
from oracle import flux_oracle as fo
from oracle.cases import Case
from tests import _image_guidance_golden as G
from tests import _lora_scale_golden as LS


@dataclass
class CallbackCase(Case):
    kind: str = "latents"          # "noop" | "latents" | "prompt" | "interrupt" | "latents_interrupt"
    edit_step: int = 1
    edit_sample: Optional[int] = None  # latents edit on this sample only (None: every sample)
    tensor_inputs: List[str] = field(default_factory=lambda: ["latents"])
    image_guidance_scale: float = 1.0
    lora_scale: float = 1.0        # joint_attention_kwargs["scale"]


CASES = {c.name: c for c in [
    CallbackCase("cb_noop", steps=4, cond_size=128, lora_rank=32, kind="noop", seed=110),
    CallbackCase("cb_edit", steps=4, cond_size=128, lora_rank=32, seed=111),
    CallbackCase("cb_prompt", steps=4, cond_size=128, lora_rank=32, kind="prompt",
                 tensor_inputs=["latents", "prompt_embeds"], seed=112),
    CallbackCase("cb_interrupt", steps=4, cond_size=128, lora_rank=32, kind="interrupt", seed=113),
    # the early-stop pattern: return edited latents and interrupt in the same step; the edit is the result
    CallbackCase("cb_edit_interrupt", steps=4, cond_size=128, lora_rank=32, kind="latents_interrupt", seed=120),
    CallbackCase("cb_ig", steps=4, cond_size=128, lora_rank=32, image_guidance_scale=1.5, seed=114),
    CallbackCase("cb_b2", steps=3, batch=2, cond_size=128, lora_rank=32, edit_sample=1, seed=115),
    CallbackCase("cb_lora07", steps=4, cond_size=128, lora_rank=32, lora_scale=0.7, seed=116),
    CallbackCase("cb_entry_a", steps=4, seed=117),
    CallbackCase("cb_deep", double=19, single=38, steps=3, cond_size=128, lora_rank=32, seed=118),
    # the headline geometry: 1024x1024 + 512x512 condition, 28 steps, an edit mid-loop
    CallbackCase("cb_1024_28", double=1, single=2, n_txt=512, height=1024, width=1024, cond_size=512, lora_rank=32,
                 steps=28, edit_step=13, seed=119),
]}

GOLDEN_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flux_golden_callback.safetensors")


def load_golden():
    from safetensors.torch import load_file
    return load_file(GOLDEN_FILE)


def _guided(case: CallbackCase) -> G.GuidedCase:
    """The case as an image-guidance case (same name and seed, so the same U_i draws)."""
    return G.GuidedCase(**{k: getattr(case, k) for k in Case.__dataclass_fields__},
                        image_guidance_scale=case.image_guidance_scale, lora_scale=case.lora_scale)


def uncond_latents(case: CallbackCase, dtype=torch.bfloat16) -> torch.Tensor:
    """U [n_steps, B, n_cond, 64] of an image-guided case (tests/_image_guidance_golden.py's draws)."""
    return G.uncond_latents(_guided(case), dtype)


def effective_scaling(case: CallbackCase) -> float:
    """The one fp32 LoRA scaling of the case over its transformer calls (1 or 2 per step)."""
    if not case.lora_rank:
        return 1.0
    calls = 2 if case.image_guidance_scale != 1.0 else 1
    return LS.effective_scaling(LS.ScaleCase(case.name, steps=calls * case.steps, lora_rank=case.lora_rank,
                                             lora_scale=case.lora_scale))


def scripted_callback(case: CallbackCase):
    """callback_on_step_end(pipe, i, t, callback_kwargs) of the case.  The edits are bf16 tensors drawn from the
    case's seed, added (latents) or swapped in (T5 states) on the device and in the dtype of the tensors they replace
    (the fp32 oracle gets the same bf16 values); a shift per channel keeps the T5 swap visible through the
    near-uniform attention of random weights."""
    def cb(pipe, i, t, kw):
        if i != case.edit_step or case.kind == "noop":
            return {}
        if case.kind.endswith("interrupt"):
            pipe._interrupt = True
            if case.kind == "interrupt":
                return {}
        g = C._gen(case, f"edit/{i}")
        if case.kind == "prompt":
            p = kw["prompt_embeds"]
            new = torch.randn(p.shape, generator=g) + 2 * torch.randn(p.shape[0], 1, p.shape[2], generator=g)
            return {"prompt_embeds": new.to(torch.bfloat16).to(p.device, p.dtype)}
        lat = kw["latents"]
        d = (0.5 * torch.randn(lat.shape, generator=g)).to(torch.bfloat16).to(lat.dtype)
        if case.edit_sample is not None:
            keep = torch.zeros(lat.shape[0], 1, 1, dtype=lat.dtype)
            keep[case.edit_sample] = 1
            d = d * keep
        return {"latents": lat + d.to(lat.device)}
    return cb


class _Pipe:
    """What the scripted callback may touch of the pipeline: the interrupt flag."""
    def __init__(self):
        self._interrupt = False

    @property
    def interrupt(self):
        return self._interrupt


def callback_denoise(model, x, case: CallbackCase, U, lora: Optional[fo.LoraSet], callback, scalar_dtype=None):
    """generate.py:217-290 with a callback (steps of the module docstring), on the oracle."""
    latents, prompt_embeds = x["latents"], x["prompt_embeds"]
    B = latents.shape[0]
    timesteps, sigmas = fo.flow_match_sigmas(case.steps, latents.shape[1])
    sd = scalar_dtype or latents.dtype
    mc = C.oracle_model_config(case)
    s = case.image_guidance_scale
    pipe = _Pipe()
    for i, t in enumerate(timesteps):
        if pipe.interrupt:
            continue
        timestep = t.expand(B).to(sd) / 1000
        guidance = torch.tensor([case.guidance]).expand(B)
        args = (latents, prompt_embeds, x["pooled"], timestep, x["img_ids"], x["txt_ids"])
        v = fo.transformer_forward(model, *args, guidance, x["cond_latents"], x["cond_ids"], mc, lora,
                                   scalar_dtype=sd)
        if s != 1.0:
            u = fo.transformer_forward(model, *args, torch.ones_like(guidance), U[i], x["cond_ids"], mc, lora,
                                       scalar_dtype=sd)
            v = u + s * (v - u)
        latents = fo.euler_step(latents, v, sigmas[i], sigmas[i + 1])
        if callback is not None:
            kw = {"latents": latents, "prompt_embeds": prompt_embeds}
            out = callback(pipe, i, t, {k: kw[k] for k in case.tensor_inputs})
            latents = out.pop("latents", latents).to(latents.dtype)
            prompt_embeds = out.pop("prompt_embeds", prompt_embeds).to(prompt_embeds.dtype)
    return latents


@torch.no_grad()
def run_oracle(case: CallbackCase, with_callback: bool = True):
    """The oracle in bf16 (the reference's arithmetic); `with_callback=False`: the same case without a callback."""
    model, lora = C.build_model(case)
    ls = fo.LoraSet(lora, effective_scaling(case)) if lora else None
    U = uncond_latents(case) if case.image_guidance_scale != 1.0 else None
    return callback_denoise(model, C.build_inputs(case), case, U, ls,
                            scripted_callback(case) if with_callback else None)


@torch.no_grad()
def fp32_oracle(case: CallbackCase):
    """fp32 arithmetic on the same bf16-valued weights, inputs and edits: the "true value"."""
    m32, l32 = C.build_model(case)
    m32 = m32.float()
    ls = fo.LoraSet({k: (a.float(), b.float()) for k, (a, b) in l32.items()}, effective_scaling(case)) if l32 else None
    x = {k: (None if v is None else (v if k in ("timestep", "guidance") else v.float()))
         for k, v in C.build_inputs(case).items()}
    U = uncond_latents(case).float() if case.image_guidance_scale != 1.0 else None
    return callback_denoise(m32, x, case, U, ls, scripted_callback(case), scalar_dtype=torch.bfloat16)
