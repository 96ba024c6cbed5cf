"""How far is the reference's bf16 graph from ITSELF when only the floating-point summation order
changes?  (VERDICT r01 weak #1d: justify replacing BASELINE.json's rtol 1e-3 / atol 1e-4.)

Runs the reference's own unmodified transformer.py / generate.py (imported from /root/reference
over oracle/shims, like make_golden.py) on the same seeded case under different CPU execution
settings — thread count (changes oneDNN's blocking / reduction split) and oneDNN on/off (a different
bf16 GEMM kernel) — and records the distances between those runs next to the distance to the fp32
evaluation.  BUILD CONTAINER ONLY.  python -m oracle.self_distance  ->  tests/golden/self_distance.json"""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle import cases as C  # noqa: E402
from oracle import make_golden, ref_loader  # noqa: E402

CASES = ["fwdA_small", "fwdB_small", "fwdA_deep", "fwdB_1024", "denoiseA_28", "denoiseB_28"]


def main():
    ns = ref_loader.load()
    gold = C.load_golden()
    out = {}
    for name in CASES:
        case = C.CASES[name]
        runs = {}
        for tag, threads, mkldnn in (("t8", os.cpu_count() or 8, True), ("t1", 1, True), ("t3", 3, True),
                                     ("t8_nomkldnn", os.cpu_count() or 8, False)):
            torch.set_num_threads(threads)
            with torch.backends.mkldnn.flags(enabled=mkldnn):
                runs[tag] = C.golden_sample(gold, name, make_golden.run_reference(ns, case).float())
        torch.set_num_threads(os.cpu_count() or 8)
        true32 = gold[name + "/fp32"].float()
        base = runs["t8"]
        rec = {"vs_fp32_mean": (base - true32).abs().mean().item(), "vs_fp32_max": (base - true32).abs().max().item()}
        for tag, r in runs.items():
            if tag == "t8":
                continue
            d = (r - base).abs()
            tol_fail = (d > 1e-4 + 1e-3 * base.abs()).float().mean().item()
            rec[tag] = {"mean": d.mean().item(), "max": d.max().item(), "bit_identical": (r == base).float().mean().item(),
                        "frac_outside_rtol1e-3_atol1e-4": tol_fail}
        out[name] = rec
        print(name, json.dumps(rec))
    with open(os.path.join(REPO, "tests", "golden", "self_distance.json"), "w") as f:
        json.dump({"generator": "oracle/self_distance.py", "torch": torch.__version__,
                   "what": "reference (unmodified transformer.py/generate.py over shims, CPU bf16) vs itself under "
                           "different thread counts / oneDNN off; base = all cores, oneDNN on", "cases": out}, f, indent=1)


if __name__ == "__main__":
    main()
