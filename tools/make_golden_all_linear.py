#!/usr/bin/env python
"""Mint tests/golden/flux_golden_all_linear.safetensors (+ .json) for the cases of tests/_all_linear_golden.py.

Needs the original project's tree (RF_REFERENCE_ROOT, default /root/reference).  For every case it wraps every
nn.Linear of the transformer in a peft-semantics LoRA layer, the way train/model.py:73-79 enumerates them for
`target_modules: "all-linear"`, runs the reference's own `tranformer_forward` / `generate` on CPU in bf16 (with
`lora_alpha / r` and `joint_attention_kwargs={"scale": s}` as tools/make_golden_lora_scale.py does), requires the
all-linear oracle to agree bit for bit, and stores a seeded sample of token rows of the bf16 output and of the
fp32-arithmetic oracle output.  It also records how far the targets outside train_flux/config.yaml:53 move the
output (the oracle with only the config.yaml:53 subset of the same factors), so a dropped term cannot hide under the
bf16 error budget.  Arguments: case names to check without writing anything."""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import cases as C  # noqa: E402
from oracle import ref_loader  # noqa: E402
from tests import _all_linear_golden as G  # noqa: E402
from tests._lora_scale_golden import effective_scaling  # noqa: E402
from tools import make_golden_lora_scale as S  # noqa: E402


def run_reference(ns, case):
    """tools/make_golden_lora_scale.run_reference with the all-linear factors: its wrap_lora wraps every module the
    factors name, so every Linear becomes a peft layer, and enable_lora gates the ones the reference names."""
    build = C.build_model
    C.build_model = G.build_model
    try:
        return S.run_reference(ns, case)
    finally:
        C.build_model = build


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
        _, full = G.build_model(case)
        gated, always = G.split(case.config(), full)
        sub = G.run_oracle(case, lora=gated)
        effect = (ora.float() - sub.float()).abs().mean().item()
        print(f"{name:18s} {len(always)} new targets  ref==oracle bit-exact: {same}  (all-linear effect: mean |d| "
              f"{effect:.4g})", flush=True)
        if not same:
            raise SystemExit(f"oracle does not reproduce the reference on case {name}")
        o32 = G.run_oracle(case, fp32=True)
        e = (ref.float() - o32).abs()
        meta[name] = {"bf16_vs_fp32_max": e.max().item(), "bf16_vs_fp32_mean": e.mean().item(),
                      "out_absmax": o32.abs().max().item(), "effective_scaling": effective_scaling(case),
                      "all_linear_effect_mean": effect}
        rows = C.golden_rows(name, ref.shape[1])
        out[name + "/rows"] = rows
        out[name + "/bf16"] = ref[:, rows].contiguous()
        out[name + "/fp32"] = o32[:, rows].contiguous()
    if only:
        print("subset run: nothing written")
        return
    save_file(out, G.GOLDEN_FILE)
    with open(G.GOLDEN_FILE.replace(".safetensors", ".json"), "w") as fjson:
        json.dump({"generator": "tools/make_golden_all_linear.py", "torch": torch.__version__, "cases": meta},
                  fjson, indent=1)
    print("wrote", G.GOLDEN_FILE)


if __name__ == "__main__":
    main()
