#!/usr/bin/env python
"""Mint tests/golden/flux_golden_latent_lora.safetensors (+ .json) for the cases of tests/_latent_lora_golden.py.

Needs the original project's tree (RF_REFERENCE_ROOT, default /root/reference).  Like oracle/make_golden.py, for
every case it runs the reference's own transformer / generate code on CPU in bf16 with `latent_lora: True`, requires
the oracle to agree bit for bit, and stores a seeded sample of token rows of the bf16 output and of the
fp32-arithmetic oracle output.  It also records how far the flag moves the output (the same case with
`latent_lora: False`), so a missing low-rank term cannot hide under the bf16 error budget.  The other golden files
are left as they are."""
import dataclasses
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import cases as C  # noqa: E402
from oracle import ref_loader  # noqa: E402
from oracle.make_golden import run_reference  # noqa: E402
from tests import _latent_lora_golden as G  # noqa: E402
from tools.make_golden_geometry import fp32_oracle  # noqa: E402


def main():
    from safetensors.torch import save_file
    ns = ref_loader.load()
    torch.set_num_threads(os.cpu_count() or 1)
    out, meta = {}, {}
    for name, case in G.CASES.items():
        assert case.model_config.get("latent_lora") is True
        ref = run_reference(ns, case)
        ora = C.run_oracle(case)
        same = torch.equal(ref, ora)
        off = C.run_oracle(dataclasses.replace(case, model_config={**case.model_config, "latent_lora": False}))
        effect = (ora.float() - off.float()).abs().mean().item()
        print(f"{name:20s} ref==oracle bit-exact: {same}  (latent_lora effect: mean |d| {effect:.4g})", flush=True)
        if not same:
            raise SystemExit(f"oracle does not reproduce the reference on case {name}")
        o32 = fp32_oracle(case)
        e = (ref.float() - o32).abs()
        meta[name] = {"bf16_vs_fp32_max": e.max().item(), "bf16_vs_fp32_mean": e.mean().item(),
                      "out_absmax": o32.abs().max().item(), "latent_lora_effect_mean": effect}
        rows = C.golden_rows(name, ref.shape[1])
        out[name + "/rows"] = rows
        out[name + "/bf16"] = ref[:, rows].contiguous()
        out[name + "/fp32"] = o32[:, rows].contiguous()
    save_file(out, G.GOLDEN_FILE)
    with open(G.GOLDEN_FILE.replace(".safetensors", ".json"), "w") as fjson:
        json.dump({"generator": "tools/make_golden_latent_lora.py", "torch": torch.__version__, "cases": meta},
                  fjson, indent=1)
    print("wrote", G.GOLDEN_FILE)


if __name__ == "__main__":
    main()
