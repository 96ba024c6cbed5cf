"""DiT golden cases whose main / condition split (n_txt + n_img) is not a multiple of 128, in the two
condition-masked attention modes (union_cond_attn=False; condition_scale != 1).  Minted by
tools/make_golden_geometry.py with the reference's own code (oracle/make_golden.py::run_reference) into
tests/golden/flux_golden_geometry.safetensors; the tile-aligned cases stay in oracle/cases.py."""
import os

from oracle.cases import Case

# 208x176 image (143 tokens) + 77 text tokens: split at 220 = 128 + 92, then a 128x128 condition (64 tokens)
CASES = {c.name: c for c in [
    Case("fwdB_ragged_mask", height=208, width=176, n_txt=77, cond_size=128, lora_rank=32, seed=40,
         model_config={"union_cond_attn": False}),
    Case("fwdB_ragged_cscale", height=208, width=176, n_txt=77, cond_size=128, lora_rank=32, seed=41,
         condition_scale=2.0),
    Case("denoiseB_ragged_mask", height=208, width=176, n_txt=77, cond_size=128, lora_rank=32, seed=42, steps=4,
         model_config={"union_cond_attn": False}),
]}

GOLDEN_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flux_golden_geometry.safetensors")


def load_golden():
    from safetensors.torch import load_file
    return load_file(GOLDEN_FILE)
