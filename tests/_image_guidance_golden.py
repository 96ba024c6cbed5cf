"""DiT golden cases with image classifier-free guidance (`generate(..., image_guidance_scale=s)`, generate.py:250-272).
Minted by tools/make_golden_image_guidance.py with the reference's own `generate()` into
tests/golden/flux_golden_image_guidance.safetensors.

Every step i of the reference's loop runs
  c = tranformer_forward(latents, t_i, guidance=g, condition_latents=C0)
  U_i = condition.encode(self, empty=True)[0]      (the real image again, condition.py:121: a fresh posterior sample)
  u = tranformer_forward(latents, t_i, guidance=ones_like(g), condition_latents=U_i)
  v = u + s * (c - u)                              (bf16 tensors, the Python scalar s taken as fp32)
then the Euler step on v.  Here U_i is seeded per case and step (`distinct_uncond`), or C0 for every step."""
import os
from dataclasses import dataclass
from typing import Optional

import torch

from oracle import cases as C
from oracle import flux_oracle as fo
from oracle.cases import Case
from tests import _lora_scale_golden as LS


@dataclass
class GuidedCase(Case):
    image_guidance_scale: float = 1.5
    distinct_uncond: bool = True   # False: U_i = C0 for every step
    lora_scale: float = 1.0        # joint_attention_kwargs["scale"]


_FULL = dict(heads=24, joint_dim=4096, pooled_dim=768, n_txt=512)

CASES = {c.name: c for c in [
    GuidedCase("ig_s15", steps=4, cond_size=128, lora_rank=32, seed=90),
    # s = 1.3: the guidance product rounds differently with a double or a bf16 scalar
    GuidedCase("ig_s13", steps=4, cond_size=128, lora_rank=32, image_guidance_scale=1.3, seed=91),
    GuidedCase("ig_neg", steps=4, cond_size=128, lora_rank=32, image_guidance_scale=-0.45, seed=92),
    GuidedCase("ig_same_u", steps=4, cond_size=128, lora_rank=32, distinct_uncond=False, seed=93),
    GuidedCase("ig_cscale", steps=4, cond_size=128, lora_rank=32, condition_scale=1.5, seed=94),
    GuidedCase("ig_mask", steps=4, cond_size=128, lora_rank=32, seed=95, model_config={"union_cond_attn": False}),
    GuidedCase("ig_ll", steps=4, cond_size=128, lora_rank=32, seed=96, model_config={"latent_lora": True}),
    # the call-level LoRA scale is scaled / unscaled around both transformer calls of every step
    GuidedCase("ig_lora07", steps=4, cond_size=128, lora_rank=32, lora_scale=0.7, seed=97),
    GuidedCase("ig_b2", steps=3, batch=2, cond_size=128, lora_rank=32, image_guidance_scale=2.0, seed=98),
    # full width with 256 condition tokens: the fused-LoRA condition group
    GuidedCase("ig_full", double=1, single=1, steps=2, cond_size=256, lora_rank=32, seed=99, **_FULL),
    # full FLUX.1-dev depth at D = 256
    GuidedCase("ig_deep", double=19, single=38, steps=3, cond_size=128, lora_rank=32, seed=100),
    # the headline geometry: 1024x1024 + 512x512 condition, 28 steps
    GuidedCase("ig_1024_28", double=1, single=2, n_txt=512, height=1024, width=1024, cond_size=512, lora_rank=32,
               steps=28, image_guidance_scale=2.0, seed=101),
]}

GOLDEN_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                           "flux_golden_image_guidance.safetensors")


def load_golden():
    from safetensors.torch import load_file
    return load_file(GOLDEN_FILE)


def uncond_latents(case: GuidedCase, dtype=torch.bfloat16, distinct: Optional[bool] = None) -> torch.Tensor:
    """U [n_steps, B, n_cond, 64]: a seeded draw per step, or C0 repeated.  Each draw carries a per-channel shift
    common to its tokens: with the near-uniform attention of random weights, token-wise independent noise averages
    out over the condition rows, and U_i would move the output no more than the bf16 error does."""
    distinct = case.distinct_uncond if distinct is None else distinct
    if not distinct:
        c0 = C.build_inputs(case, dtype)["cond_latents"]
        return c0[None].expand(case.steps, *c0.shape).contiguous()
    out = []
    for i in range(case.steps):
        g = C._gen(case, f"uncond/{i}")
        u = torch.randn(case.batch, case.n_cond, 64, generator=g) + 4 * torch.randn(case.batch, 1, 64, generator=g)
        out.append(u.to(dtype))
    return torch.stack(out)


def effective_scaling(case: GuidedCase) -> float:
    """The one fp32 LoRA scaling of the case: peft scales and unscales around each of the 2 calls per step."""
    probe = LS.ScaleCase(case.name, steps=2 * case.steps, lora_rank=case.lora_rank, lora_scale=case.lora_scale)
    return LS.effective_scaling(probe)


def guided_denoise(model, x, case: GuidedCase, U, lora: Optional[fo.LoraSet], s: float, scalar_dtype=None):
    """generate.py:217-276 with image_guidance_scale s (steps 1-5 of the module docstring), on the oracle."""
    latents = x["latents"]
    B = latents.shape[0]
    timesteps, sigmas = fo.flow_match_sigmas(case.steps, latents.shape[1])
    sd = scalar_dtype or latents.dtype
    mc = C.oracle_model_config(case)
    for i, t in enumerate(timesteps):
        timestep = t.expand(B).to(sd) / 1000
        guidance = torch.tensor([case.guidance]).expand(B)
        args = (latents, x["prompt_embeds"], x["pooled"], timestep, x["img_ids"], x["txt_ids"])
        v = fo.transformer_forward(model, *args, guidance, x["cond_latents"], x["cond_ids"], mc, lora,
                                   scalar_dtype=sd)
        if s != 1.0:
            u = fo.transformer_forward(model, *args, torch.ones_like(guidance), U[i], x["cond_ids"], mc, lora,
                                       scalar_dtype=sd)
            v = u + s * (v - u)
        latents = fo.euler_step(latents, v, sigmas[i], sigmas[i + 1])
    return latents


@torch.no_grad()
def run_oracle(case: GuidedCase, s: Optional[float] = None, distinct: Optional[bool] = None):
    """The oracle in bf16 (the reference's arithmetic); `s` / `distinct` override the case's."""
    model, lora = C.build_model(case)
    ls = fo.LoraSet(lora, effective_scaling(case)) if lora else None
    return guided_denoise(model, C.build_inputs(case), case, uncond_latents(case, distinct=distinct), ls,
                          case.image_guidance_scale if s is None else s)


@torch.no_grad()
def fp32_oracle(case: GuidedCase):
    """fp32 arithmetic on the same bf16-valued weights and inputs: the "true value"."""
    m32, l32 = C.build_model(case)
    m32 = m32.float()
    ls = fo.LoraSet({k: (a.float(), b.float()) for k, (a, b) in l32.items()}, effective_scaling(case)) if l32 else None
    x = {k: (None if v is None else (v if k in ("timestep", "guidance") else v.float()))
         for k, v in C.build_inputs(case).items()}
    return guided_denoise(m32, x, case, uncond_latents(case).float(), ls, case.image_guidance_scale,
                          scalar_dtype=torch.bfloat16)
