#!/usr/bin/env python
"""Cost of per-step callbacks on the headline entry B loop: 1024x1024 + 512x512 condition, 28 steps, reference-exact
LoRA (rank 32), random weights, full FLUX.1-dev depth.  Times `generate(output_type="latent")` three ways, alternating
within one run (REPEATS rounds, default 3): no callback (the whole-loop rf_dit_denoise), a no-op callback, and a
callback that reads the latents on the device (a mean, kept on the device).  The callback paths run the step-wise
session (rf_dit_denoise_begin / rf_dit_denoise_step).  Prints one JSON line with the median ms per call and per step of
each, the overhead of each callback path over the plain loop, the card's name and its power limit read in this run.

Env: LAYERS=double,single (default 19,38), STEPS (default 28), REPEATS (default 3)."""
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from reflectionflow_b200.config import FluxDiTConfig  # noqa: E402
from reflectionflow_b200.pipeline import B200FluxPipeline, Condition, generate  # noqa: E402
from reflectionflow_b200.tts.reflectionflow import synthetic_lora  # noqa: E402

dev = torch.device("cuda:0")
layers = os.environ.get("LAYERS", "19,38").split(",")
cfg = FluxDiTConfig(num_layers=int(layers[0]), num_single_layers=int(layers[1]))
steps = int(os.environ.get("STEPS", "28"))
repeats = int(os.environ.get("REPEATS", "3"))
pipe = B200FluxPipeline.from_synthetic(cfg, seed=0, device=dev, lora_rank=32)
pipe.transformer.load_lora(synthetic_lora(cfg, rank=32), mode="exact")
g = torch.Generator().manual_seed(0)
lat = torch.randn(1, 4096, 64, generator=g).to(torch.bfloat16)
txt = torch.randn(1, 512, 4096, generator=g).to(torch.bfloat16)
pool = torch.randn(1, 768, generator=g).to(torch.bfloat16)
cond = Condition("cot", latents=torch.randn(1, 1024, 64, generator=g).to(torch.bfloat16), position_delta=[0, -32])
sums = []


def noop(p, i, t, kw):
    return {}


def read_latents(p, i, t, kw):
    sums.append(kw["latents"].float().mean())  # stays on the device: no synchronisation
    return {}


VARIANTS = {"none": None, "noop": noop, "read_latents": read_latents}


def run(cb):
    return generate(pipe, conditions=[cond], model_config={"union_cond_attn": True}, default_lora=True,
                    prompt_embeds=txt, pooled_prompt_embeds=pool, latents=lat, height=1024, width=1024,
                    num_inference_steps=steps, output_type="latent", callback_on_step_end=cb).images


outs = {k: run(cb) for k, cb in VARIANTS.items()}  # warm-up: capture, allocations
assert torch.equal(outs["none"], outs["noop"]) and torch.equal(outs["none"], outs["read_latents"])
torch.cuda.synchronize()
times = {k: [] for k in VARIANTS}
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for _ in range(repeats):
    for k, cb in VARIANTS.items():
        e0.record()
        run(cb)
        e1.record()
        torch.cuda.synchronize()
        times[k].append(e0.elapsed_time(e1))
        sums.clear()
try:
    power_limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                 capture_output=True, text=True, timeout=30).stdout.strip()
except Exception:
    power_limit = "unknown"
med = {k: statistics.median(v) for k, v in times.items()}
print(json.dumps({"workload": "entry B 1024^2 + 512^2 cond, exact LoRA r32", "layers": layers, "steps": steps,
                  "repeats": repeats, "ms_per_call": med, "ms_per_step": {k: v / steps for k, v in med.items()},
                  "all_ms": times,
                  "overhead_pct": {k: 100 * (med[k] / med["none"] - 1) for k in ("noop", "read_latents")},
                  "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit}))
