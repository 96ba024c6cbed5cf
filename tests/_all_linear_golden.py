"""DiT golden cases with an adapter on every Linear of FluxTransformer2DModel: what train/model.py:73-80 trains with
`target_modules: "all-linear"`, and what most diffusers-format FLUX LoRAs cover (the text stream, ff.net.0.proj).
Minted by tools/make_golden_all_linear.py with the reference's own code into
tests/golden/flux_golden_all_linear.safetensors.

The oracle of these cases is oracle/flux_oracle.py with the Linears outside train_flux/config.yaml:53 wrapped in
peft's arithmetic (`AlwaysLora`).  No enable_lora block names those modules, so every call applies them; the
config.yaml:53 targets keep going through `LoraSet.linear` with their enable_lora gating.  The factors of the
config.yaml:53 subset are those of `fo.make_lora_weights` (seeded per module name), so each case also says how far
the new targets move the output: oracle(all-linear) against oracle(the config.yaml:53 subset of the same factors).

The geometries pick which LoRA groups of the CUDA step take the fused low-rank k-block (>= 128 rows) and which keep
the unfused fallback (< 128 rows): 77 text tokens put the text stream on the fallback."""
import math
import os
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import cases as C
from oracle import flux_oracle as fo
from tests._lora_scale_golden import ScaleCase, effective_scaling

_FULL = dict(heads=24, joint_dim=4096, pooled_dim=768, n_txt=512)

CASES = {c.name: c for c in [
    # entry A without latent_lora: only the always-on targets act (text stream, embedders, ff.net.0.proj, final
    # layer); 128 text tokens: fused text groups
    ScaleCase("fwdA_al_t128", lora_rank=32, seed=90),
    # 77 text tokens: the text groups take the unfused fallback
    ScaleCase("fwdA_al_t77", n_txt=77, lora_rank=32, seed=91),
    ScaleCase("fwdB_al_small", cond_size=128, lora_rank=32, seed=92),
    # full width (D = 3072, T5 4096, 512 text tokens, 256 condition tokens)
    ScaleCase("fwdB_al_full", double=1, single=1, cond_size=256, lora_rank=32, seed=93, **_FULL),
    # the headline geometry: 1024x1024 + 512x512 condition
    ScaleCase("fwdB_al_1024", double=2, single=2, n_txt=512, height=1024, width=1024, cond_size=512, lora_rank=32,
              seed=94),
    # full FLUX.1-dev depth at D = 256: per-layer offsets of the new targets and of their modulation terms
    ScaleCase("fwdB_al_deep", double=19, single=38, cond_size=128, lora_rank=32, seed=95),
    # latent_lora with rank 128, alpha != r and a call scale
    ScaleCase("fwdB_al_ll_r128", cond_size=256, lora_rank=128, lora_alpha=64, lora_scale=0.8, seed=96,
              model_config={"latent_lora": True}),
    ScaleCase("fwdB_al_mask", cond_size=128, lora_rank=32, seed=97, model_config={"union_cond_attn": False}),
    # the embedder terms batched over all 28 steps of the loop, with a call scale
    ScaleCase("denoiseB_al_28_s", double=2, single=2, steps=28, cond_size=128, lora_rank=32, lora_scale=0.7,
              seed=98),
    ScaleCase("denoiseA_al_4", steps=4, lora_rank=32, seed=99),
]}

GOLDEN_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flux_golden_all_linear.safetensors")


def load_golden():
    from safetensors.torch import load_file
    return load_file(GOLDEN_FILE)


def all_linear_modules(model: nn.Module) -> List[str]:
    """Every nn.Linear of the transformer by name, as train/model.py:73-79 enumerates them for peft."""
    return sorted(name for name, m in model.named_modules() if isinstance(m, nn.Linear))


def make_lora_weights(model: nn.Module, rank: int, seed: int,
                      dtype=torch.bfloat16) -> Dict[str, Tuple[torch.Tensor, torch.Tensor]]:
    """Seeded factors {module: (A [r, in], B [out, r])} on every Linear, drawn like fo.make_lora_weights: one
    generator per module name, so the config.yaml:53 modules get exactly that function's factors."""
    mods = dict(model.named_modules())
    out = {}
    for name in all_linear_modules(model):
        lin = mods[name]
        g = torch.Generator().manual_seed(fo._name_seed(name + ".lora", seed))
        A = torch.randn(rank, lin.in_features, generator=g) / math.sqrt(lin.in_features)
        B = torch.randn(lin.out_features, rank, generator=g) * (0.5 / math.sqrt(rank))
        out[name] = (A.to(dtype), B.to(dtype))
    return out


def build_model(case: ScaleCase, dtype=torch.bfloat16):
    """(oracle model, all-linear factors) of a case; the drop-in for oracle.cases.build_model."""
    model = fo.FluxTransformer2DModel(case.config())
    fo.init_weights_(model, seed=case.seed, dtype=dtype)
    model.eval()
    return model, make_lora_weights(model, case.lora_rank, case.seed + 100, dtype)


class AlwaysLora(nn.Module):
    """peft's LoRA Linear for a module that no enable_lora block names: y = base(x) + lora_B(lora_A(x)) * scaling on
    every call."""

    def __init__(self, base: nn.Linear, A: torch.Tensor, B: torch.Tensor, scaling: float):
        super().__init__()
        self.base, self.A, self.B, self.scaling = base, A, B, scaling

    def forward(self, x):
        return self.base(x) + F.linear(F.linear(x, self.A.to(x.dtype)), self.B.to(x.dtype)) * self.scaling


def split(cfg: fo.FluxConfig, lora: Dict) -> Tuple[Dict, Dict]:
    """(the config.yaml:53 targets, the others)"""
    gated = set(fo.lora_target_modules(cfg))
    return ({k: v for k, v in lora.items() if k in gated}, {k: v for k, v in lora.items() if k not in gated})


def _wrap_always(model: nn.Module, lora: Dict, scaling: float) -> None:
    for name, (A, B) in lora.items():
        parent_name, _, attr = name.rpartition(".")
        parent = model.get_submodule(parent_name) if parent_name else model
        if attr.isdigit():
            parent[int(attr)] = AlwaysLora(parent[int(attr)], A, B, scaling)
        else:
            setattr(parent, attr, AlwaysLora(getattr(parent, attr), A, B, scaling))


@torch.no_grad()
def run_oracle(case: ScaleCase, lora: Optional[Dict] = None, scaling: Optional[float] = None, fp32: bool = False):
    """The oracle with the adapter `lora` (default: the case's all-linear factors; any subset of them works) at the
    case's effective scaling.  fp32: fp32 arithmetic on the same bf16-valued weights and inputs (the "true value")."""
    model, full = build_model(case)
    lora = full if lora is None else lora
    s = effective_scaling(case) if scaling is None else scaling
    x = C.build_inputs(case)
    if fp32:
        model = model.float()
        lora = {k: (a.float(), b.float()) for k, (a, b) in lora.items()}
        x = {k: (None if v is None else (v if k in ("timestep", "guidance") else v.float())) for k, v in x.items()}
    gated, always = split(case.config(), lora)
    _wrap_always(model, always, s)
    ls = fo.LoraSet(gated, s) if gated else None
    mc = C.oracle_model_config(case)
    sd = torch.bfloat16 if fp32 else None
    if case.steps:
        return fo.denoise(model, x["latents"], x["prompt_embeds"], x["pooled"], case.steps, case.guidance,
                          x["img_ids"], x["txt_ids"], x["cond_latents"], x["cond_ids"], mc, ls, scalar_dtype=sd)
    return fo.transformer_forward(model, x["latents"], x["prompt_embeds"], x["pooled"], x["timestep"], x["img_ids"],
                                  x["txt_ids"], x["guidance"], x["cond_latents"], x["cond_ids"], mc, ls,
                                  scalar_dtype=sd)
