"""DiT golden cases with a scaled LoRA: `lora_alpha != r` (peft scaling = lora_alpha / r) and a call-level
`joint_attention_kwargs={"scale": s}` (diffusers' LoRA strength), with adapter ranks up to 128.  Minted by
tools/make_golden_lora_scale.py with the reference's own code into tests/golden/flux_golden_lora_scale.safetensors.

The effective scaling of a target is lora_alpha / r * s, formed in double as peft does (`scaling *= scale`) and
rounded once to fp32 where torch multiplies the bf16 low-rank term by it.  Every alpha / r below is exact in fp32.

The geometries pick fused (>= 128 rows) and fallback (< 128 rows) LoRA groups, one and two 64-deep low-rank k-blocks
(rank <= 64 / rank 65..128) and a rank that is zero-padded (96 -> 128)."""
import os
from dataclasses import dataclass
from typing import List, Optional

import torch

from oracle import cases as C
from oracle import flux_oracle as fo
from oracle.cases import Case


@dataclass
class ScaleCase(Case):
    lora_alpha: Optional[float] = None  # None: lora_alpha = r (scaling 1)
    lora_scale: float = 1.0             # joint_attention_kwargs["scale"]

    @property
    def alpha_over_r(self) -> float:
        return 1.0 if self.lora_alpha is None else self.lora_alpha / self.lora_rank


_FULL = dict(heads=24, joint_dim=4096, pooled_dim=768, n_txt=512)

CASES = {c.name: c for c in [
    # call scale; 64 condition tokens: the condition group takes the unfused fallback
    ScaleCase("fwdB_s075", cond_size=128, lora_rank=32, lora_scale=0.75, seed=70),
    # alpha != r; 256 condition tokens: fused condition group
    ScaleCase("fwdB_c256_a16", cond_size=256, lora_rank=32, lora_alpha=16, seed=71),
    ScaleCase("fwdB_neg", cond_size=256, lora_rank=32, lora_scale=-0.5, seed=72),
    # full width, rank 128: two low-rank k-blocks and the q|k|v sections of the stacked T
    ScaleCase("fwdB_full_r128", double=1, single=1, cond_size=256, lora_rank=128, seed=73, **_FULL),
    # rank 96 zero-padded to 128
    ScaleCase("fwdB_full_r96", double=1, single=1, cond_size=256, lora_rank=96, lora_alpha=48, lora_scale=1.5,
              seed=74, **_FULL),
    # latent_lora: image / text groups, x_embedder and the adaLN terms, all scaled
    ScaleCase("fwdB_ll_r128", cond_size=128, lora_rank=128, lora_alpha=64, lora_scale=0.8, seed=75,
              model_config={"latent_lora": True}),
    # the headline geometry: 1024x1024 + 512x512 condition
    ScaleCase("fwdB_1024_r128", double=2, single=2, n_txt=512, height=1024, width=1024, cond_size=512,
              lora_rank=128, lora_scale=0.6, seed=76),
    # full FLUX.1-dev depth at D = 256: per-layer offsets of the 128-wide LoRA storage
    ScaleCase("fwdB_deep_r128", double=19, single=38, cond_size=128, lora_rank=128, lora_alpha=256, seed=77),
    # masked mode: the image rows do not attend to the condition rows, so the adapter acts through latent_lora
    ScaleCase("fwdB_mask_s", cond_size=128, lora_rank=64, lora_alpha=32, lora_scale=1.25, seed=78,
              model_config={"union_cond_attn": False, "latent_lora": True}),
    # the scale / unscale sequence around each of the 28 steps of a denoise loop
    ScaleCase("denoiseB_28_s", double=2, single=2, steps=28, cond_size=128, lora_rank=32, lora_scale=0.7, seed=79),
    # text-to-image with a scaled adapter on the image
    ScaleCase("denoiseA_ll_r128_s", steps=4, lora_rank=128, lora_scale=0.5, seed=80,
              model_config={"latent_lora": True}),
]}

GOLDEN_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flux_golden_lora_scale.safetensors")


def load_golden():
    from safetensors.torch import load_file
    return load_file(GOLDEN_FILE)


def reference_scalings(case: ScaleCase) -> List[float]:
    """The double `scaling` of a target during each transformer call of the case, following the reference: peft
    sets alpha / r at load; every call multiplies by s (`scale_layer`) and divides by it afterwards (`unscale_layer`;
    s == 0 resets through `set_scale(adapter, 1.0)`), so (alpha/r * s) / s carries over to the next call."""
    r = case.lora_rank
    alpha = case.alpha_over_r * r
    s = case.lora_scale
    scaling = alpha / r
    out = []
    for _ in range(max(case.steps, 1)):
        if s != 1:
            scaling *= s
        out.append(scaling)
        if s == 0:
            scaling = 1.0 * alpha / r
        elif s != 1:
            scaling /= s
    return out


def effective_scaling(case: ScaleCase) -> float:
    """The one fp32 scaling the case applies; fails if the reference's per-call values differ in fp32."""
    f32 = {torch.tensor(v, dtype=torch.float32).item() for v in reference_scalings(case)}
    assert len(f32) == 1, f"{case.name}: the per-call scaling differs in fp32: {sorted(f32)}"
    return f32.pop()


def _run(case: ScaleCase, model, lora, x, scaling, scalar_dtype=None):
    ls = fo.LoraSet(lora, scaling) if lora else None
    mc = C.oracle_model_config(case)
    if case.steps:
        return fo.denoise(model, x["latents"], x["prompt_embeds"], x["pooled"], case.steps, case.guidance,
                          x["img_ids"], x["txt_ids"], x["cond_latents"], x["cond_ids"], mc, ls,
                          scalar_dtype=scalar_dtype)
    return fo.transformer_forward(model, x["latents"], x["prompt_embeds"], x["pooled"], x["timestep"],
                                  x["img_ids"], x["txt_ids"], x["guidance"], x["cond_latents"], x["cond_ids"],
                                  mc, ls, scalar_dtype=scalar_dtype)


@torch.no_grad()
def run_oracle(case: ScaleCase, scaling: Optional[float] = None):
    """The oracle in bf16 with the case's effective scaling (or `scaling`)."""
    model, lora = C.build_model(case)
    return _run(case, model, lora, C.build_inputs(case), effective_scaling(case) if scaling is None else scaling)


@torch.no_grad()
def fp32_oracle(case: ScaleCase):
    """fp32 arithmetic on the same bf16-valued weights and inputs: the "true value"."""
    m32, l32 = C.build_model(case)
    m32 = m32.float()
    l32 = {k: (a.float(), b.float()) for k, (a, b) in l32.items()}
    x = {k: (None if v is None else (v if k in ("timestep", "guidance") else v.float()))
         for k, v in C.build_inputs(case).items()}
    return _run(case, m32, l32, x, effective_scaling(case), scalar_dtype=torch.bfloat16)
