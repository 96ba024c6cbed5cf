"""Seeded parity cases shared by oracle/make_golden.py (reference vs oracle, build container) and
tests/ (oracle vs golden on CPU; CUDA path vs oracle/golden on the GPU).  TEST INFRASTRUCTURE.

Every tensor is a pure function of (case name, seed): nothing but the expected outputs needs to
be stored in tests/golden/."""
from __future__ import annotations

import os
import zlib
from dataclasses import dataclass, field
from typing import Dict, Optional

import torch

from . import flux_oracle as fo


@dataclass
class Case:
    name: str
    heads: int = 2
    double: int = 1
    single: int = 1
    joint_dim: int = 128
    pooled_dim: int = 64
    n_txt: int = 128
    height: int = 256          # image size in pixels -> (h/16)*(w/16) tokens
    width: int = 256
    cond_size: int = 0         # condition image size in pixels (0 = entry A)
    lora_rank: int = 0
    steps: int = 0             # > 0: denoise-loop case
    batch: int = 1
    model_config: Dict = field(default_factory=dict)
    condition_scale: float = 1.0
    sigma: float = 0.75        # timestep (already / 1000) of single-forward cases
    guidance: float = 3.5
    seed: int = 0

    @property
    def n_img(self):
        return (self.height // 16) * (self.width // 16)

    @property
    def n_cond(self):
        return (self.cond_size // 16) ** 2

    def config(self) -> fo.FluxConfig:
        return fo.FluxConfig(num_layers=self.double, num_single_layers=self.single,
                             num_attention_heads=self.heads, joint_attention_dim=self.joint_dim,
                             pooled_projection_dim=self.pooled_dim)


CASES = {c.name: c for c in [
    Case("fwdA_small"),
    Case("fwdA_small_b2", batch=2, seed=3),
    Case("fwdB_small", cond_size=128, lora_rank=32, seed=1),
    Case("fwdB_small_nolora", cond_size=128, seed=2),
    Case("fwdB_small_mask", cond_size=128, lora_rank=32, seed=4,
         model_config={"union_cond_attn": False}),
    Case("fwdB_small_cscale", cond_size=128, lora_rank=32, seed=5, condition_scale=2.0),
    Case("fwdA_ragged", height=208, width=176, n_txt=77, seed=6),
    Case("fwdA_full", heads=24, double=1, single=1, joint_dim=4096, pooled_dim=768, n_txt=512,
         seed=7),
    Case("fwdB_full", heads=24, double=1, single=1, joint_dim=4096, pooled_dim=768, n_txt=512,
         cond_size=128, lora_rank=32, seed=8),
    Case("denoiseA_small", steps=4, seed=9),
    Case("denoiseB_small", steps=4, cond_size=128, lora_rank=32, seed=10),
    Case("denoiseA_full", heads=24, double=1, single=1, joint_dim=4096, pooled_dim=768, n_txt=512,
         steps=4, seed=11),
    # ---- round 2: depth, geometry and step-count coverage (VERDICT r01 "weak" #1)
    # full FLUX.1-dev depth (19 double + 38 single) at D = 256: per-layer offsets into the stacked
    # modulation table / weight packs and 57-block error growth
    Case("fwdA_deep", double=19, single=38, seed=12),
    Case("fwdB_deep", double=19, single=38, cond_size=128, lora_rank=32, seed=13),
    # more than one block of each kind at full width (D = 3072, joint 4096, 512 text tokens)
    Case("fwdB_mid", heads=24, double=2, single=3, joint_dim=4096, pooled_dim=768, n_txt=512,
         cond_size=128, lora_rank=32, seed=14),
    # the headline geometries: 1024x1024 -> N = 4608 (entry A) and + 512x512 condition -> N = 5632
    Case("fwdA_1024", double=2, single=2, n_txt=512, height=1024, width=1024, seed=15),
    Case("fwdB_1024", double=2, single=2, n_txt=512, height=1024, width=1024, cond_size=512,
         lora_rank=32, seed=16),
    Case("fwdB_1024_mask", double=1, single=2, n_txt=512, height=1024, width=1024, cond_size=512,
         lora_rank=32, seed=17, model_config={"union_cond_attn": False}),
    Case("fwdB_1024_cscale", double=2, single=1, n_txt=512, height=1024, width=1024, cond_size=512,
         lora_rank=32, seed=18, condition_scale=1.5),
    # the metric's 28-step schedule
    Case("denoiseA_28", double=2, single=2, steps=28, seed=19),
    Case("denoiseB_28", double=2, single=2, steps=28, cond_size=128, lora_rank=32, seed=20),
    Case("denoiseB_1024_28", double=1, single=2, n_txt=512, height=1024, width=1024, cond_size=512,
         lora_rank=32, steps=28, seed=21),
    Case("denoiseB_deep_28", double=19, single=38, steps=28, cond_size=128, lora_rank=32, seed=22),
    # full width with >= 128 condition tokens: the fused-LoRA condition GEMMs (gemm2_lora_launch)
    Case("fwdB_full_c256", heads=24, double=1, single=1, joint_dim=4096, pooled_dim=768, n_txt=512,
         cond_size=256, lora_rank=32, seed=23),
]}


def _gen(case: Case, tag: str) -> torch.Generator:
    return torch.Generator().manual_seed(fo._name_seed(case.name + "/" + tag, case.seed))


def build_model(case: Case, dtype=torch.bfloat16):
    model = fo.FluxTransformer2DModel(case.config())
    fo.init_weights_(model, seed=case.seed, dtype=dtype)
    model.eval()
    lora = None
    if case.lora_rank:
        lora = fo.make_lora_weights(model, case.config(), rank=case.lora_rank, seed=case.seed + 100,
                                    dtype=dtype)
    return model, lora


def build_inputs(case: Case, dtype=torch.bfloat16) -> Dict[str, Optional[torch.Tensor]]:
    B = case.batch
    d = {}
    d["latents"] = torch.randn(B, case.n_img, 64, generator=_gen(case, "latents")).to(dtype)
    d["prompt_embeds"] = torch.randn(B, case.n_txt, case.joint_dim, generator=_gen(case, "t5")).to(dtype)
    d["pooled"] = torch.randn(B, case.pooled_dim, generator=_gen(case, "clip")).to(dtype)
    d["img_ids"] = fo.prepare_latent_image_ids(case.height // 16, case.width // 16, dtype)
    d["txt_ids"] = torch.zeros(case.n_txt, 3, dtype=dtype)
    d["timestep"] = torch.full((B,), case.sigma).to(dtype)
    d["guidance"] = torch.full((B,), case.guidance, dtype=torch.float32)
    if case.cond_size:
        d["cond_latents"] = torch.randn(B, case.n_cond, 64, generator=_gen(case, "cond")).to(dtype)
        d["cond_ids"] = fo.condition_ids(case.cond_size, (0, -(case.cond_size // 16)), dtype)
    else:
        d["cond_latents"] = None
        d["cond_ids"] = None
    return d


def oracle_model_config(case: Case) -> Dict:
    mc = dict(case.model_config)
    if case.condition_scale != 1.0:
        mc["_c_factor"] = case.condition_scale
    return mc


@torch.no_grad()
def run_oracle(case: Case, dtype=torch.bfloat16, model=None, lora=None):
    if model is None:
        model, lora = build_model(case, dtype)
    x = build_inputs(case, dtype)
    ls = fo.LoraSet(lora, 1.0) if lora else None
    mc = oracle_model_config(case)
    if case.steps:
        return fo.denoise(model, x["latents"], x["prompt_embeds"], x["pooled"], case.steps,
                          case.guidance, x["img_ids"], x["txt_ids"], x["cond_latents"],
                          x["cond_ids"], mc, ls)
    return fo.transformer_forward(model, x["latents"], x["prompt_embeds"], x["pooled"],
                                  x["timestep"], x["img_ids"], x["txt_ids"], x["guidance"],
                                  x["cond_latents"], x["cond_ids"], mc, ls)


# ---- stored golden outputs: a seeded sample of GOLDEN_ROWS token rows per case keeps the file small; every
# comparison against the golden runs on the same rows (`golden_sample`)
GOLDEN_ROWS = 64
GOLDEN_FILE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                           "flux_golden.safetensors")


def golden_rows(name: str, n_tok: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    return torch.randperm(n_tok, generator=g)[:min(GOLDEN_ROWS, n_tok)].sort().values


def golden_sample(gold: Dict[str, torch.Tensor], name: str, t: torch.Tensor) -> torch.Tensor:
    """the golden rows of case `name` of an output [batch, n_tok, 64]"""
    return t[:, gold[name + "/rows"]]


def load_golden() -> Dict[str, torch.Tensor]:
    from safetensors.torch import load_file
    return load_file(GOLDEN_FILE)
