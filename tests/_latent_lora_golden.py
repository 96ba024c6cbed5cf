"""DiT golden cases with `latent_lora: True`: the LoRA acts on the image tokens (and, in the single-stream blocks, on
the text tokens too), not only on the condition tokens.  Minted by tools/make_golden_latent_lora.py with the
reference's own code (oracle/make_golden.py::run_reference) into tests/golden/flux_golden_latent_lora.safetensors.

The geometries pick which LoRA groups of the CUDA step take the fused low-rank k-block (>= 128 rows) and which keep
the unfused fallback (< 128 rows)."""
import os

from oracle.cases import Case

_LL = {"latent_lora": True}
_FULL = dict(heads=24, joint_dim=4096, pooled_dim=768, n_txt=512)

CASES = {c.name: c for c in [
    # entry A: text-to-image with a LoRA on the image (256 image tokens: fused image group)
    Case("fwdA_ll_small", lora_rank=32, seed=50, model_config=dict(_LL)),
    # 256 image tokens fused, 64 condition tokens on the unfused fallback
    Case("fwdB_ll_small", cond_size=128, lora_rank=32, seed=51, model_config=dict(_LL)),
    # 128x176 image = 88 tokens: the double-block image group falls back, the single-block txt+img group
    # (77 + 88 = 165 rows) is fused
    Case("fwdB_ll_tinyimg", height=128, width=176, n_txt=77, cond_size=128, lora_rank=32, seed=52,
         model_config=dict(_LL)),
    # full width (D = 3072), 512 text tokens, 256 condition tokens: every LoRA group fused
    Case("fwdB_ll_full", double=1, single=1, cond_size=256, lora_rank=32, seed=53, model_config=dict(_LL),
         **_FULL),
    # the headline geometry: 1024x1024 + 512x512 condition
    Case("fwdB_ll_1024", double=2, single=2, n_txt=512, height=1024, width=1024, cond_size=512, lora_rank=32,
         seed=54, model_config=dict(_LL)),
    # full FLUX.1-dev depth at D = 256: per-layer offsets of the modulation LoRA terms
    Case("fwdB_ll_deep", double=19, single=38, cond_size=128, lora_rank=32, seed=55, model_config=dict(_LL)),
    Case("fwdB_ll_mask", cond_size=128, lora_rank=32, seed=56,
         model_config={"latent_lora": True, "union_cond_attn": False}),
    Case("denoiseA_ll_small", steps=4, lora_rank=32, seed=57, model_config=dict(_LL)),
    Case("denoiseB_ll_28", double=2, single=2, steps=28, cond_size=128, lora_rank=32, seed=58,
         model_config=dict(_LL)),
]}

GOLDEN_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flux_golden_latent_lora.safetensors")


def load_golden():
    from safetensors.torch import load_file
    return load_file(GOLDEN_FILE)
