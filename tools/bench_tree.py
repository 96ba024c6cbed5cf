#!/usr/bin/env python
"""Headline workload: FLUX-dev 1024x1024, 28 steps x 8 candidates x 4 reflection
rounds (entry B: 512x512 condition stream + LoRA), candidates sharded over the ranks, one all-gather of
score records + one of candidate latents per round, VAE decode / resize / encode of every parent, stub
verifier + reflector.  Prints one JSON line (rank 0).  torchrun-compatible."""
import json, os, sys, time
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from reflectionflow_b200 import _lib as L
from reflectionflow_b200.tts import reflectionflow as RF, search as S
from reflectionflow_b200.tts.dist import DistCtx
from reflectionflow_b200.tts.utils import get_noises
from reflectionflow_b200.tts.verifiers import Candidate, StubReflector, StubVerifier

ctx = DistCtx.from_env()
layers = os.environ.get("LAYERS", "19,38")
steps = int(os.environ.get("STEPS", "28"))
branch, rounds = int(os.environ.get("BRANCH", "8")), int(os.environ.get("ROUNDS", "4"))
cfg = json.load(open(os.path.join(os.path.dirname(RF.__file__), "configs", "headline_tree_flux_dev.json")))
cfg["search_args"].update(search_branch=branch, search_rounds=rounds)
cfg["pipeline_args"]["num_inference_steps"] = steps


class A:
    synthetic, layers_ = True, layers
A.layers = layers
A.lora_mode = os.environ.get("LORA_MODE", "exact")
A.text_encoders = os.environ.get("TEXT", "native")  # T5-XXL + CLIP-L of every candidate prompt run on the device
pipe = RF.build_pipeline(cfg, A, ctx)
torch.manual_seed(0)
g = torch.Generator().manual_seed(7)
parents = [Candidate(f"r0/{i}.png", i, latents=torch.randn(1, 4096, 64, generator=g).to(torch.bfloat16).to(ctx.device))
           for i in range(branch)]
out = os.environ.get("OUT", "/tmp/tree_out")
dirs = {k: os.path.join(out, k) for k in ("last", "best", "bestround", "mid")}
if ctx.rank == 0:
    for d in dirs.values():
        os.makedirs(d, exist_ok=True)
ctx.barrier()


def gen(pipe_, **kw):  # generate() defaults to 28 steps; honour STEPS for short runs
    return RF._generate(pipe_, num_inference_steps=steps, **kw)


def run(n_rounds, parents):
    chains, upd, refl = {}, ["a photo of a cat"] * branch, [""] * branch
    for rnd in range(1, n_rounds + 1):
        noises = get_noises(S.MAX_SEED, branch, 1024, 1024)
        dp = RF.sample(noises, "a photo of a cat", upd, refl, rnd, pipe, branch, out, cfg, dirs["last"],
                       dirs["best"], dirs["bestround"], parents, dirs["mid"], n_rounds, chains,
                       verifier=StubVerifier("nvila"), reflector=StubReflector(), ctx=ctx, generate_fn=gen,
                       defer_saves=True)
        parents, chains = dp["generated"], dp["chains"]
        upd, refl = dp["refined_prompt"], dp["reflections"]
    RF.flush_saves()  # every artefact on disk before the clock stops
    return parents


import builtins
_print = builtins.print
builtins.print = lambda *a, **k: None  # silence the per-phase prints of sample()
run(1, parents)  # warm-up round (graph capture, workspaces)
torch.cuda.synchronize(); ctx.barrier()
l0 = L.load().rf_launch_count()
t0 = time.time()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
run(rounds, parents)
e1.record(); torch.cuda.synchronize(); ctx.barrier()
wall = time.time() - t0
ms = e0.elapsed_time(e1)
builtins.print = _print
if ctx.world > 1:
    import torch.distributed as dist
    t = torch.tensor([ms], device=ctx.device); dist.all_reduce(t, op=dist.ReduceOp.MAX); ms = t.item()
n_steps = steps * branch * rounds
if ctx.rank == 0:
    print(json.dumps({"workload": f"{steps}-step x {branch}-cand x {rounds}-round reflection tree, 1024x1024, cond 512x512, "
                                  f"LoRA {A.lora_mode}, " "VAE decode+resize+encode per parent, PNG+latent artefacts written, text encoders: " + A.text_encoders,
                      "n_gpus": ctx.world, "layers": layers, "denoise_steps": n_steps, "images": branch * rounds,
                      "seconds": ms / 1e3, "wall_seconds": wall, "denoise_steps_per_s": n_steps / (ms / 1e3),
                      "images_per_s": branch * rounds / (ms / 1e3),
                      "gpu_launches_rank0": int(L.load().rf_launch_count() - l0)}))
if ctx.world > 1:
    import torch.distributed as dist
    dist.destroy_process_group()
