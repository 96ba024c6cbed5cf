#!/usr/bin/env python
"""Mint tests/golden/flux_golden_geometry.safetensors (+ .json) for the cases of tests/_geometry_golden.py.

Needs the original project's tree (RF_REFERENCE_ROOT, default /root/reference).  Like oracle/make_golden.py, for
every case it runs the reference's own transformer / generate code on CPU in bf16, requires the oracle to agree
bit for bit, and stores a seeded sample of token rows of the bf16 output and of the fp32-arithmetic oracle
output.  The main golden file is left as it is."""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import cases as C  # noqa: E402
from oracle import flux_oracle as fo  # noqa: E402
from oracle import ref_loader  # noqa: E402
from oracle.make_golden import run_reference  # noqa: E402
from tests import _geometry_golden as G  # noqa: E402


def fp32_oracle(case):
    m32, l32 = C.build_model(case, torch.bfloat16)
    m32 = m32.float()
    l32 = {k: (a.float(), b.float()) for k, (a, b) in l32.items()} if l32 else None
    x = C.build_inputs(case, torch.bfloat16)
    ls = fo.LoraSet(l32, 1.0) if l32 else None
    mc = C.oracle_model_config(case)
    f = lambda t: None if t is None else t.float()  # noqa: E731
    if case.steps:
        return fo.denoise(m32, f(x["latents"]), f(x["prompt_embeds"]), f(x["pooled"]), case.steps, case.guidance,
                          f(x["img_ids"]), f(x["txt_ids"]), f(x["cond_latents"]), f(x["cond_ids"]), mc, ls,
                          scalar_dtype=torch.bfloat16)
    return fo.transformer_forward(m32, f(x["latents"]), f(x["prompt_embeds"]), f(x["pooled"]), x["timestep"],
                                  f(x["img_ids"]), f(x["txt_ids"]), x["guidance"], f(x["cond_latents"]),
                                  f(x["cond_ids"]), mc, ls, scalar_dtype=torch.bfloat16)


def main():
    from safetensors.torch import save_file
    ns = ref_loader.load()
    torch.set_num_threads(os.cpu_count() or 1)
    out, meta = {}, {}
    for name, case in G.CASES.items():
        ref = run_reference(ns, case)
        ora = C.run_oracle(case)
        print(f"{name:22s} n_main {case.n_txt + case.n_img} ref==oracle bit-exact: {torch.equal(ref, ora)}")
        if not torch.equal(ref, ora):
            raise SystemExit(f"oracle does not reproduce the reference on case {name}")
        o32 = fp32_oracle(case)
        e = (ref.float() - o32).abs()
        meta[name] = {"bf16_vs_fp32_max": e.max().item(), "bf16_vs_fp32_mean": e.mean().item(),
                      "out_absmax": o32.abs().max().item()}
        rows = C.golden_rows(name, ref.shape[1])
        out[name + "/rows"] = rows
        out[name + "/bf16"] = ref[:, rows].contiguous()
        out[name + "/fp32"] = o32[:, rows].contiguous()
    save_file(out, G.GOLDEN_FILE)
    with open(G.GOLDEN_FILE.replace(".safetensors", ".json"), "w") as fjson:
        json.dump({"generator": "tools/make_golden_geometry.py", "torch": torch.__version__, "cases": meta}, fjson,
                  indent=1)
    print("wrote", G.GOLDEN_FILE)


if __name__ == "__main__":
    main()
