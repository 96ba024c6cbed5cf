#!/usr/bin/env python
"""bench.py — denoise-steps/s and images/s of the FLUX.1-dev 1024x1024 reflection tree
(28 steps x 8 candidates x 4 rounds) on N H100s of one node.

  python bench.py [--gpus N] [--steps K] [--warmup W]          product arm (CUDA kernels)
  python bench.py ... --dump-outputs DIR                        also write the final latents of the
                                                                timed headline call to DIR/latents.npy
  python bench.py --impl reference ...                          reference arm: the reference's CPU
                                                                path (oracle port) on host cores

One "step" = one denoise step of one candidate on the HEADLINE path, entry B of the reference
(tts_reflectionflow.py -> generate() -> tranformer_forward): DiT forward over 512 text + 4096 image
+ 1024 condition tokens (5632), rank-32 LoRA on the condition tokens, + the flow-match Euler update.

The ONE JSON line carries
  value / ms_per_step   K headline steps per rank, inputs resident in HBM (weak scaling: every rank
                        runs its own candidate, as a search round does)
  tree                  the whole tree as ONE timed call: 8 candidates x 4 rounds x K-step denoise,
                        T5-XXL + CLIP-L encode of every candidate prompt, VAE decode -> PIL-exact resize ->
                        VAE encode of every parent, both all-gathers per round, PNG + latent artefacts
                        flushed — candidates sharded over the N ranks (STRONG scaling); images_per_sec
                        comes from here
  entry_a               the condition-free step (configs[1], 4608 tokens) as a secondary number
  e2e                   the headline steps through generate() with pinned-HOST inputs and host read-back
  roofline / kernels    per-kernel split of one eager headline forward, dominant kernel vs the
                        measured tensor peak
  gpu_eager_baseline    the SAME step run the way the reference runs it on a GPU: the oracle's torch
                        graph on CUDA (cuBLAS + SDPA, eager), same box, same run
  cpu_baseline          the oracle port on the host cores (bounded sample), whose output is also
                        compared with the CUDA blocks on the same weights (SURVEY §8d)
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

STEPS_PER_IMAGE = 28
H = W = 1024
COND = 512
N_TXT = 512
N_IMG = (H // 16) * (W // 16)
N_COND = (COND // 16) ** 2
D_MODEL = 3072
BRANCH, ROUNDS = 8, 4


def algorithmic_tflop(n_tok: int, layers: int = 57, d: int = D_MODEL) -> float:
    """SURVEY.md §8(d): 57 * 24 D^2 N (GEMM) + 57 * 4 N^2 D (attention), 2 FLOP/MAC."""
    return (layers * 24 * d * d * n_tok + layers * 4 * n_tok * n_tok * d) / 1e12


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        j = json.load(open(p))
        return {"tflops_burst": j["bf16_tflops"], "tflops_sustained": j["bf16_tflops_sustained"],
                "hbm_gbs": j["hbm_gbs"], "source": "measured"}
    # NVIDIA H100 SXM data sheet (dense bf16, HBM3), not measured: the sustained rate under a power cap is lower
    return {"tflops_burst": 989.0, "tflops_sustained": 989.0, "hbm_gbs": 3350.0,
            "source": "fallback (H100 SXM data sheet)"}


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region."""

    def __init__(self, gpu_index: int):
        self.rows = []
        self.proc = None
        self.gpu = gpu_index
        self.t = None

    def start(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.gpu}", f"--query-gpu={q}",
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except Exception:
            self.proc = None
            return
        self.t = threading.Thread(target=self._read, daemon=True)
        self.t.start()

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons, pw = [], [], set(), []
        for r in self.rows:
            f = [x.strip() for x in r.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx.append(float(f[1])); pw.append(float(f[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown",
                                "sw_power_cap"), f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no samples"]}
        busy = sorted(s for s, p in zip(sm, pw) if p > 300) or sorted(sm)
        return {"sm_mhz": busy[len(busy) // 2], "sm_max_mhz": max(mx), "reasons": sorted(reasons),
                "samples": len(sm), "power_w_max": max(pw)}


# ------------------------------------------------------------------------------------------------
# CPU arm: the reference's own arithmetic (oracle port of block.py / transformer.py over restated
# diffusers leaves) on the host cores
# ------------------------------------------------------------------------------------------------
def physical_cores() -> int:
    try:
        import psutil
        n = psutil.cpu_count(logical=False)
        if n:
            return int(n)
    except Exception:
        pass
    return os.cpu_count() or 1


def cpu_reference_leg(samples: int, warmup: int, want_output: bool = False):
    """A full headline step is 95 TFLOP over a 23.8 GB model, so each timed "step" of this arm is a
    BOUNDED SAMPLE: one forward of a ONE double + ONE single block FLUX.1-dev-width model at the real
    headline geometry (N = 5632: 512 txt + 4096 img + 1024 cond, LoRA on the cond tokens), blocks
    timed individually; step time = 19 x t_double + 38 x t_single (embedders / final layer are
    < 0.1 % of the FLOPs).  >= 2 warm-ups, >= 3 samples, MEDIAN; threads = physical cores."""
    import torch
    from oracle import flux_oracle as fo
    cores = physical_cores()
    torch.set_num_threads(cores)
    samples, warmup = max(3, samples), max(2, warmup)
    cfg = fo.FluxConfig.tiny_depth(1, 1)
    model = fo.FluxTransformer2DModel(cfg)
    fo.init_weights_(model, seed=0)
    model.eval()
    lora = fo.make_lora_weights(model, cfg, rank=32, seed=1)
    x = parity_inputs()
    t_blocks = {"d": [], "s": []}
    orig_d, orig_s = fo.double_block, fo.single_block

    def timed(fn, key):
        def wrap(*a, **k):
            t0 = time.perf_counter()
            r = fn(*a, **k)
            t_blocks[key].append(time.perf_counter() - t0)
            return r
        return wrap
    fo.double_block, fo.single_block = timed(orig_d, "d"), timed(orig_s, "s")
    out = None
    try:
        with torch.no_grad():
            for it in range(warmup + samples):
                out = fo.transformer_forward(model, x["latents"], x["prompt_embeds"], x["pooled"], x["timestep"],
                                             x["img_ids"], x["txt_ids"], x["guidance"], x["cond_latents"],
                                             x["cond_ids"], {}, fo.LoraSet(lora, 1.0))
    finally:
        fo.double_block, fo.single_block = orig_d, orig_s
    td_all, ts_all = t_blocks["d"][warmup:], t_blocks["s"][warmup:]
    td, ts = statistics.median(td_all), statistics.median(ts_all)
    step_s = 19 * td + 38 * ts
    spread = max(max(td_all) / min(td_all), max(ts_all) / min(ts_all))
    par = torch.__config__.parallel_info().strip().splitlines()
    par = "; ".join(l.strip() for l in par if any(k in l for k in ("get_num_threads", "OMP_NUM", "MKL_NUM", "ATen parallel backend", "mkldnn")))
    leg = {"value": 1.0 / step_s, "unit": "denoise-steps/s", "cores": cores, "kind": "port",
           "sample": (f"1 double + 1 single FLUX.1-dev block at the headline geometry N=5632 (cond stream + LoRA), bf16, "
                      f"torch CPU: median of {len(td_all)} samples after {warmup} warm-ups: double {td:.2f} s, single {ts:.2f} s "
                      f"(max/min over samples {spread:.2f}); step = 19 x double + 38 x single = {step_s:.1f} s (extrapolated)"),
           "ms_per_step": step_s * 1e3, "threads": cores, "logical_cpus": os.cpu_count(), "parallel_info": par,
           "t_double_s": td_all, "t_single_s": ts_all}
    if want_output:
        leg["_output"], leg["_model"], leg["_lora"] = out, model, lora
    return leg


def parity_inputs():
    """Seeded inputs of the headline geometry shared by the CPU leg and its CUDA comparison."""
    import torch
    from oracle import flux_oracle as fo
    g = torch.Generator().manual_seed(0)
    bf = torch.bfloat16
    return {"latents": torch.randn(1, N_IMG, 64, generator=g).to(bf),
            "prompt_embeds": torch.randn(1, N_TXT, 4096, generator=g).to(bf),
            "pooled": torch.randn(1, 768, generator=g).to(bf),
            "cond_latents": torch.randn(1, N_COND, 64, generator=g).to(bf),
            "img_ids": fo.prepare_latent_image_ids(H // 16, W // 16, bf),
            "txt_ids": torch.zeros(N_TXT, 3, dtype=bf),
            "cond_ids": fo.condition_ids(COND, (0, -(COND // 16)), bf),
            "timestep": torch.full((1,), 0.75).to(bf), "guidance": torch.full((1,), 3.5)}


def cuda_parity_of_cpu_leg(leg, dev):
    """SURVEY §8(d): the timed CPU output doubles as the parity reference — same weights, same inputs
    through the CUDA blocks (1 double + 1 single at full width, headline geometry, exact LoRA)."""
    import torch
    from reflectionflow_b200.transformer import B200FluxTransformer2DModel, tranformer_forward
    model, lora, ref = leg.pop("_model"), leg.pop("_lora"), leg.pop("_output")
    from oracle import flux_oracle as fo
    m = B200FluxTransformer2DModel(fo.FluxConfig.tiny_depth(1, 1), lora_rank=32, device=dev)
    m.load_state_dict(model.state_dict())
    m.load_lora(lora, mode="exact")
    x = parity_inputs()
    out = tranformer_forward(m, x["cond_latents"], x["cond_ids"], None, {}, 0, hidden_states=x["latents"],
                             encoder_hidden_states=x["prompt_embeds"], pooled_projections=x["pooled"],
                             timestep=x["timestep"], img_ids=x["img_ids"], txt_ids=x["txt_ids"],
                             guidance=x["guidance"], return_dict=False)[0]
    torch.cuda.synchronize(dev)
    d = (out.cpu().float() - ref.float()).abs()
    m.close()
    par = {"what": "CUDA 1+1-block forward vs the timed CPU output, same weights/inputs, N=5632, exact LoRA",
           "mean_abs_diff": d.mean().item(), "max_abs_diff": d.max().item(),
           "bit_identical": (out.cpu() == ref).float().mean().item(), "ref_absmax": ref.float().abs().max().item()}
    if not (d.mean().item() < 6e-3 and d.max().item() < 0.15):
        raise RuntimeError(f"CUDA blocks deviate from the CPU reference leg: {par}")
    return par


_REAL_STDOUT = None


def _quiet_stdout():
    """Libraries (NCCL's version banner, ...) write to fd 1; the contract is ONE JSON line on stdout.
    Route fd 1 to stderr for the whole run and keep the real stdout for the final line."""
    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)


def _emit(line: dict):
    out = _REAL_STDOUT or sys.stdout
    out.write(json.dumps(line) + "\n")
    out.flush()


def log(*a):
    print("[bench]", *a, file=sys.stderr, flush=True)


# ------------------------------------------------------------------------------------------------
# the tree: tts_reflectionflow.py's loop on this repo's pipeline, one timed call
# ------------------------------------------------------------------------------------------------
def run_tree(pipe, ctx, steps: int, branch: int, rounds: int, out_dir: str, cfg_json: dict):
    import builtins
    import torch
    from reflectionflow_b200.tts import reflectionflow as RF, search as S
    from reflectionflow_b200.tts.utils import get_noises
    from reflectionflow_b200.tts.verifiers import Candidate, StubReflector, StubVerifier
    cfg = json.loads(json.dumps(cfg_json))
    cfg["search_args"].update(search_branch=branch, search_rounds=rounds)
    cfg["pipeline_args"]["num_inference_steps"] = steps
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(7)
    parents = [Candidate(f"r0/{i}.png", i, latents=torch.randn(1, N_IMG, 64, generator=g).to(torch.bfloat16).to(ctx.device))
               for i in range(branch)]
    dirs = {k: os.path.join(out_dir, k) for k in ("last", "best", "bestround", "mid")}
    if ctx.rank == 0:
        for d in dirs.values():
            os.makedirs(d, exist_ok=True)
    ctx.barrier()

    def gen(pipe_, **kw):
        return RF._generate(pipe_, num_inference_steps=steps, **kw)
    _print = builtins.print
    builtins.print = lambda *a, **k: None  # silence the per-phase prints of sample()
    try:
        chains, upd, refl = {}, ["a photo of a cat"] * branch, [""] * branch
        for rnd in range(1, rounds + 1):
            noises = get_noises(S.MAX_SEED, branch, H, W)
            dp = RF.sample(noises, "a photo of a cat", upd, refl, rnd, pipe, branch, out_dir, cfg, dirs["last"],
                           dirs["best"], dirs["bestround"], parents, dirs["mid"], rounds, chains,
                           verifier=StubVerifier("nvila"), reflector=StubReflector(), ctx=ctx, generate_fn=gen,
                           defer_saves=True)
            parents, chains = dp["generated"], dp["chains"]
            upd, refl = dp["refined_prompt"], dp["reflections"]
        RF.flush_saves()  # every artefact on disk before the clock stops
    finally:
        builtins.print = _print
    return parents


def main():
    _quiet_stdout()
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=STEPS_PER_IMAGE)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--lora-mode", default="exact", choices=["exact", "merged"],
                    help="exact = peft's unfused low-rank arithmetic (what the reference runs); merged = fuse_lora")
    ap.add_argument("--no-tree", action="store_true")
    ap.add_argument("--no-eager", action="store_true")
    ap.add_argument("--no-text", action="store_true", help="tree with hash text embeddings instead of native T5/CLIP")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--layers", default="19,38", help="double,single layer counts (debug only)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the final latents of the last timed headline call as DIR/latents.npy (float32)")
    args = ap.parse_args()
    K, Wm = max(args.steps, 1), max(args.warmup, 0)
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    config = {"workload": "headline: tts_reflectionflow.py entry B — FLUX.1-dev DiT 1024x1024 + 512x512 condition stream "
                          "(512 txt + 4096 img + 1024 cond = 5632 tokens), rank-32 LoRA on the condition tokens "
                          f"(lora_mode={args.lora_mode}), guidance 3.5, batch 1, 1 candidate per GPU; `tree` = 8 candidates x 4 "
                          "rounds x --steps denoise steps as one timed call",
              "parallelism": f"candidate-sharded x{args.gpus} (replicated weights)",
              "l2": "inputs larger than L2: every step streams 23.8 GB of weights (H100 L2 = 50 MB)",
              "weights": "random-init (seeded), FLUX.1-dev architecture, 11.9 B params bf16 + rank-32 LoRA"}

    if args.impl == "reference":
        if rank != 0:
            return
        leg = cpu_reference_leg(min(K, 5), min(Wm, 3))
        line = {"impl": "reference", "metric": "denoise-steps/sec", "value": leg["value"],
                "unit": "denoise-steps/s", "n_gpus": args.gpus, "steps": K, "warmup": Wm,
                "ms_per_step": leg["ms_per_step"], "higher_is_better": True, "scaling": "weak",
                "vs_baseline": None, "dtype": "bf16", "data": "synthetic", "config": config,
                "cpu_baseline": {k: leg[k] for k in ("value", "unit", "cores", "kind", "sample", "threads",
                                                     "logical_cpus", "parallel_info", "t_double_s", "t_single_s")},
                "e2e": {"value": leg["value"], "unit": "denoise-steps/s", "h2d_bytes_per_step": 0,
                        "d2h_bytes_per_step": 0},
                "gpu_launches": 0}
        _emit(line)
        return

    import torch
    import torch.distributed as dist
    if not torch.cuda.is_available():
        _emit({"error": "no CUDA device: the product arm has no CPU fallback"})
        sys.exit(2)
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    from reflectionflow_b200 import _lib as L
    from reflectionflow_b200.pipeline import Condition, flow_match_schedule, generate
    from reflectionflow_b200.transformer import tranformer_forward
    from reflectionflow_b200.tts import reflectionflow as RF
    from reflectionflow_b200.tts.dist import DistCtx
    from reflectionflow_b200.tts.search import gather_scores, stub_verifier_score

    ctx = DistCtx(rank, world, dev)
    tree_cfg = json.load(open(os.path.join(os.path.dirname(RF.__file__), "configs", "headline_tree_flux_dev.json")))

    class A:
        synthetic, layers = True, args.layers
        text_encoders = "hash" if args.no_text else "native"
        lora_mode = args.lora_mode
    t_setup = time.time()
    pipe = RF.build_pipeline(tree_cfg, A, ctx)
    model = pipe.transformer
    cfg = model.cfg
    nl, ns = cfg.num_layers, cfg.num_single_layers
    lib = L.load()
    torch.cuda.synchronize()
    log(f"pipeline ready in {time.time() - t_setup:.1f} s")
    mc = tree_cfg.get("model", {})

    # synthetic inputs of the named shape (seeded per rank = per candidate)
    g = torch.Generator().manual_seed(1000 + rank)
    bf = torch.bfloat16
    lat_host = torch.randn(1, N_IMG, 64, generator=g).to(bf).pin_memory()
    txt_host = torch.randn(1, N_TXT, cfg.joint_attention_dim, generator=g).to(bf).pin_memory()
    pool_host = torch.randn(1, cfg.pooled_projection_dim, generator=g).to(bf).pin_memory()
    cond_host = torch.randn(1, N_COND, 64, generator=g).to(bf).pin_memory()
    lat, txt, pool, cond = lat_host.to(dev), txt_host.to(dev), pool_host.to(dev), cond_host.to(dev)
    img_ids = pipe._prepare_latent_image_ids(1, H // 16, W // 16, dev, bf)
    txt_ids = torch.zeros(N_TXT, 3, dtype=bf, device=dev)
    _, cond_ids, _ = Condition("cot", latents=cond, position_delta=[0, -(COND // 16)]).encode(pipe)

    def sched(n):
        ts, sig = flow_match_schedule(max(n, 1), N_IMG)  # the mu-shifted n-step schedule
        return (ts.to(bf) / 1000), sig

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(ms):
        if world > 1:
            t = torch.tensor([ms], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            return t.item()
        return ms

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed_denoise(n, use_cond):
        """n steps, inputs resident in HBM, + the round's score exchange; device-timed, max over ranks"""
        t_n, s_n = sched(n)
        barrier()
        e0.record()
        final = model.denoise(lat, txt, pool, t_n, s_n, 3.5, img_ids, txt_ids,
                              cond if use_cond else None, cond_ids if use_cond else None, mc)
        score = stub_verifier_score(final)
        if world > 1:
            gather_scores(score, rank, world, dev)  # the round's one exchange step (NCCL all-gather)
        e1.record()
        barrier()
        return max_over_ranks(e0.elapsed_time(e1)), final

    # ---- headline step (entry B): warm-up (captures the step graph), then K timed steps
    if Wm:
        timed_denoise(Wm, True)
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
        time.sleep(0.3)
    launches0 = lib.rf_launch_count()
    ms, final = timed_denoise(K, True)
    launches = lib.rf_launch_count() - launches0
    clocks = sampler.stop() if rank == 0 else None
    log(f"headline: {ms / K:.2f} ms/step")
    if args.dump_outputs and rank == 0:
        import numpy as np
        os.makedirs(args.dump_outputs, exist_ok=True)
        # [1, 4096, 64] packed latents: what model.denoise() hands its caller (1 MB as float32)
        np.save(os.path.join(args.dump_outputs, "latents.npy"), final.float().cpu().numpy())

    # ---- e2e: the public API call (generate(), entry B) with HOST inputs and a host read-back
    def e2e_call(n):
        c = Condition("cot", latents=cond_host, position_delta=[0, -(COND // 16)])
        out = generate(pipe, conditions=[c], model_config=mc, default_lora=True, prompt_embeds=txt_host,
                       pooled_prompt_embeds=pool_host, latents=lat_host, num_inference_steps=n,
                       guidance_scale=3.5, height=H, width=W, output_type="latent")
        sc = stub_verifier_score(out.images)
        if world > 1:
            gather_scores(sc, rank, world, dev)
        sc.cpu()
        return out.images.cpu()
    e2e_call(1)
    barrier()
    e0.record()
    res = e2e_call(K)
    e1.record()
    barrier()
    ms_e2e = max_over_ranks(e0.elapsed_time(e1))
    h2d = (lat_host.numel() + txt_host.numel() + pool_host.numel() + cond_host.numel()) * 2
    d2h = res.numel() * 2 + 8

    # ---- e2e at the reference's PER-STEP call granularity (tranformer_forward, transformer.py:47):
    # every step copies its latents host->device from pinned memory and reads the prediction back
    t_k, _ = sched(K)
    gd = torch.tensor([3.5], device=dev)
    pred_host = torch.empty(1, N_IMG, 64, dtype=bf).pin_memory()

    def step_call(i):
        x = lat_host.to(dev, non_blocking=True)
        out = tranformer_forward(model, cond, cond_ids, None, mc, 0, hidden_states=x, encoder_hidden_states=txt,
                                 pooled_projections=pool, timestep=t_k[i:i + 1].to(dev), img_ids=img_ids,
                                 txt_ids=txt_ids, guidance=gd, return_dict=False)[0]
        pred_host.copy_(out, non_blocking=True)
    step_call(0)
    barrier()
    e0.record()
    for i in range(K):
        step_call(i)
    e1.record()
    barrier()
    ms_fwd = max_over_ranks(e0.elapsed_time(e1))

    # ---- per-kernel breakdown of one eager headline forward (CUDA events around every launch), taken
    # hot: a 6-step denoise runs immediately before, so kernels are timed in the same power-capped
    # state as the timed region and compare against the SUSTAINED peak
    prof = None
    if rank == 0:
        t_h, s_h = sched(6)
        model.denoise(lat, txt, pool, t_h, s_h, 3.5, img_ids, txt_ids, cond, cond_ids, mc)
        L.profile_start()
        tranformer_forward(model, cond, cond_ids, None, mc, 0, hidden_states=lat, encoder_hidden_states=txt,
                           pooled_projections=pool, timestep=torch.tensor([1.0], dtype=bf), img_ids=img_ids,
                           txt_ids=txt_ids, guidance=torch.tensor([3.5]), return_dict=False)
        prof = L.profile_stop()

    # ---- entry A (configs[1]: no condition stream, 4608 tokens) as a secondary number
    if Wm:
        timed_denoise(min(Wm, 3), False)
    ms_a, _ = timed_denoise(K, False)
    log(f"entry A: {ms_a / K:.2f} ms/step")

    # ---- the other LoRA arithmetic as a secondary number: merged (peft fuse_lora: bf16(W + BA) on the condition
    # tokens) when the headline is exact, and vice versa
    other_mode = "merged" if args.lora_mode == "exact" else "exact"
    model.load_lora(RF.synthetic_lora(cfg, seed=1), mode=other_mode)
    timed_denoise(3, True)
    ms_other, _ = timed_denoise(K, True)
    model.load_lora(RF.synthetic_lora(cfg, seed=1), mode=args.lora_mode)
    timed_denoise(2, True)  # back to the headline mode (re-captures the step graph) before the tree
    log(f"lora_mode={other_mode}: {ms_other / K:.2f} ms/step")

    # ---- VAE decode of the final latent (the per-image tail: generate.py:302-307), device-timed
    for _ in range(2):
        pipe.vae.decode_packed(final, H, W, "u8")
    barrier()
    e0.record()
    for _ in range(3):
        pipe.vae.decode_packed(final, H, W, "u8")
    e1.record()
    barrier()
    ms_vae = e0.elapsed_time(e1) / 3

    # ---- text encoders of one candidate prompt (T5-XXL 512 tokens + CLIP-L 77 tokens: generate.py:148-161)
    ms_text = None
    enc = getattr(pipe, "text_encoders", None)
    if enc is not None:
        gi = torch.Generator().manual_seed(5)
        ids_t5 = torch.randint(0, 32000, (1, N_TXT), generator=gi).pin_memory()
        ids_clip = torch.randint(3, 49000, (1, 77), generator=gi)
        ids_clip[:, -1] = 49407
        ids_clip = ids_clip.pin_memory()
        for _ in range(2):
            enc.t5_encode(ids_t5); enc.clip_encode(ids_clip)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(3):
            enc.t5_encode(ids_t5); enc.clip_encode(ids_clip)
        e1.record()
        torch.cuda.synchronize()
        ms_text = e0.elapsed_time(e1) / 3

    # ---- the tree: 8 candidates x 4 rounds x K steps as ONE timed call, candidates sharded over ranks
    tree = None
    if not args.no_tree:
        import shutil
        import tempfile
        out_dir = tempfile.mkdtemp(prefix=f"rf_tree_r{rank}_") if world == 1 else os.path.join(
            tempfile.gettempdir(), f"rf_tree_{os.environ.get('MASTER_PORT', '0')}")
        run_tree(pipe, ctx, 2, max(world, 2), 1, os.path.join(out_dir, "warm"), tree_cfg)  # warm-up round
        barrier()
        l0 = lib.rf_launch_count()
        t0 = time.time()
        e0.record()
        run_tree(pipe, ctx, K, BRANCH, ROUNDS, os.path.join(out_dir, "run"), tree_cfg)
        e1.record()
        barrier()
        wall = time.time() - t0
        ms_tree = max_over_ranks(e0.elapsed_time(e1))
        n_steps = K * BRANCH * ROUNDS
        tree_tflop = n_steps * algorithmic_tflop(N_TXT + N_IMG + N_COND, nl + ns)
        n_png = 0
        if rank == 0:
            n_png = sum(f.endswith(".png") for f in os.listdir(os.path.join(out_dir, "run", "mid")))
        tree = {"workload": f"{K}-step x {BRANCH}-candidate x {ROUNDS}-round reflection tree, 1024x1024, condition 512x512, "
                            f"LoRA {args.lora_mode}; per candidate: T5-XXL + CLIP-L prompt encode ({A.text_encoders}), parent VAE decode -> "
                            "PIL-exact resize -> VAE encode, denoise, VAE decode, stub verifier; per round: 2 record all-gathers + 1 "
                            "latent all-gather; PNG + latent artefacts written and flushed inside the clock",
                "scaling": "strong", "n_gpus": world, "denoise_steps": n_steps, "images": BRANCH * ROUNDS,
                "seconds": ms_tree / 1e3, "wall_seconds": wall, "denoise_steps_per_s": n_steps / (ms_tree / 1e3),
                "images_per_s": BRANCH * ROUNDS / (ms_tree / 1e3), "num_inference_steps": K,
                "tflops_achieved_aggregate": tree_tflop / (ms_tree / 1e3),
                "frac_of_n_x_sustained_peak": tree_tflop / (ms_tree / 1e3) / (world * peaks()["tflops_sustained"]),
                "pure_denoise_seconds_at_measured_step": (n_steps / world) * (ms / K) / 1e3,
                "midimg_pngs_written": n_png, "gpu_launches_rank0": int(lib.rf_launch_count() - l0)}
        log(f"tree: {ms_tree / 1e3:.2f} s")
        if rank == 0:
            shutil.rmtree(out_dir, ignore_errors=True)

    # ---- the step the way the reference executes it on a GPU: the oracle's torch graph on CUDA
    # (eager: cuBLAS GEMMs + SDPA + elementwise kernels), same geometry, same box, same run
    eager = None
    if rank == 0 and not args.no_eager:
        try:
            eager = gpu_eager_leg(dev, nl, ns, min(K, 6))
            log(f"eager torch: {eager['ms_per_step']:.1f} ms/step")
        except Exception as e:  # noqa: BLE001 - reported in the line, never silently dropped
            eager = {"unavailable": f"{type(e).__name__}: {e}"}

    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    if rank != 0:
        return

    pk = peaks()
    n_tok = N_TXT + N_IMG + N_COND
    step_tflop = algorithmic_tflop(n_tok, nl + ns)
    step_tflop_a = algorithmic_tflop(N_TXT + N_IMG, nl + ns)
    steps_per_s = args.gpus * K / (ms / 1e3)
    # the LoRA down-projections run on a forked stream, on a few reserved SMs, beside the other streams' GEMMs
    # (csrc/dit.cu): their launch durations overlap those GEMMs and are not part of the step's critical path
    forked = {"lora_down"} if (args.lora_mode == "exact" and os.environ.get("RF_SIDE_STREAM", "1") != "0") else set()
    tot_ms = sum(v["ms"] for k, v in prof.items() if k not in forked)
    dom_name, dom = max(((k, v) for k, v in prof.items() if k not in forked), key=lambda kv: kv[1]["ms"])
    ach = dom["flops"] / (dom["ms"] / 1e3) / 1e12
    roofline = {"kernel": dom_name, "bound": "tensor", "achieved": ach,
                "peak": pk["tflops_sustained"], "unit": "TFLOP/s", "frac": ach / pk["tflops_sustained"],
                "peak_source": pk["source"],
                "algorithmic_bytes_per_launch": round(dom["bytes"] / dom["launches"]),
                "launches_per_step": dom["launches"], "avg_launch_ms": dom["ms"] / dom["launches"],
                "share_of_step": dom["ms"] / tot_ms,
                "how": "CUDA events around every launch of one eager headline forward inside this run"}
    kernels = {k: {"launches": v["launches"], "ms": round(v["ms"], 4),
                   "share": None if k in forked else round(v["ms"] / tot_ms, 4),
                   "tflops": round(v["flops"] / (v["ms"] / 1e3) / 1e12, 1) if v["flops"] else None,
                   "gbs": round(v["bytes"] / (v["ms"] / 1e3) / 1e9, 1)} for k, v in prof.items()}
    for k in forked & set(kernels):
        kernels[k]["note"] = ("forked stream: 4 CTAs on reserved SMs, concurrent with the image + text GEMM of the "
                              "same layer; its duration is hidden, not a share of the step")
    line = {"metric": "denoise-steps/sec", "value": steps_per_s, "unit": "denoise-steps/s",
            "n_gpus": args.gpus, "steps": K, "warmup": Wm, "ms_per_step": ms / K,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
            "data": "synthetic", "config": config, "lora_mode": args.lora_mode,
            "step_tflop": step_tflop,
            "step_tflops_achieved": step_tflop / (ms / K / 1e3),
            "step_frac_of_tensor_peak": step_tflop / (ms / K / 1e3) / pk["tflops_sustained"],
            "images_per_sec": tree["images_per_s"] if tree else None,
            "images_note": "32 images of the tree / the tree's ONE timed call (text encode, condition encode, denoise, decode, "
                           "artefacts, exchanges all inside)",
            "tree": tree,
            "entry_a": {"workload": "configs[1]: FLUX.1-dev 1024x1024, no condition stream (4608 tokens)",
                        "ms_per_step": ms_a / K, "value": args.gpus * K / (ms_a / 1e3), "step_tflop": step_tflop_a,
                        "step_tflops_achieved": step_tflop_a / (ms_a / K / 1e3),
                        "step_frac_of_tensor_peak": step_tflop_a / (ms_a / K / 1e3) / pk["tflops_sustained"]},
            "other_lora_mode": {"lora_mode": other_mode, "ms_per_step": ms_other / K,
                                "value": args.gpus * K / (ms_other / 1e3),
                                "note": "exact = peft's unfused y = bf16(bf16(xW^T+b) + bf16(bf16(xA^T)B^T)) (what the reference "
                                        "runs, lora_controller.py:5-42); merged = peft fuse_lora semantics bf16(W + BA) — one "
                                        "rounding of the merged weight instead of three of the low-rank path; both pass the same "
                                        "error budget against the fp32 evaluation (tests/test_gpu_dit.py)"},
            "vae_decode_ms": ms_vae, "text_encode_ms": ms_text,
            "e2e": {"value": args.gpus * K / (ms_e2e / 1e3), "unit": "denoise-steps/s",
                    "h2d_bytes_per_step": h2d / K, "d2h_bytes_per_step": d2h / K,
                    "api": "generate(pipe, conditions=[Condition('cot', latents=<pinned host>)], prompt_embeds=<pinned host>, "
                           "latents=<pinned host>, output_type='latent') -> score -> .cpu()",
                    "per_step_forward_api": {"value": args.gpus * K / (ms_fwd / 1e3), "unit": "denoise-steps/s",
                                             "h2d_bytes_per_step": lat_host.numel() * 2 + 2,
                                             "d2h_bytes_per_step": lat_host.numel() * 2,
                                             "api": "tranformer_forward(hidden_states=<pinned host>.to(dev), condition stream) -> "
                                                    "pinned host, once per step (no CUDA graph)"},
                    "note": "same work as `value` plus the copies (< 5 MB per K-step call)"},
            "gpu_launches": int(launches), "roofline": roofline, "kernels": kernels, "clocks": clocks,
            "gpu_eager_baseline": eager}
    if eager and "ms_per_step" in eager:
        line["speedup_vs_gpu_eager"] = eager["ms_per_step"] / (ms / K)
    if not args.no_cpu_baseline and args.gpus == 1:  # the CPU baseline is timed at N=1 only
        leg = cpu_reference_leg(3, 2, want_output=True)
        parity = cuda_parity_of_cpu_leg(leg, dev)
        line["cpu_baseline"] = {k: leg[k] for k in ("value", "unit", "cores", "kind", "sample", "threads",
                                                    "logical_cpus", "parallel_info")}
        line["cpu_baseline"]["parity_vs_cuda"] = parity
    _emit(line)


def gpu_eager_leg(dev, nl: int, ns: int, steps: int):
    """oracle/flux_oracle.py's graph (= the reference's block.py / transformer.py arithmetic over
    restated diffusers leaves) executed by stock torch CUDA ops, bf16, eager — what
    tts_reflectionflow.py:500 `pipe.to("cuda")` runs.  Timing only (weights: torch default init)."""
    import torch
    from oracle import flux_oracle as fo
    bf = torch.bfloat16
    cfg = fo.FluxConfig.tiny_depth(nl, ns)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(bf)
    try:
        with torch.device(dev):
            model = fo.FluxTransformer2DModel(cfg)
    finally:
        torch.set_default_dtype(prev)
    model.eval()
    g = torch.Generator(device=dev).manual_seed(3)
    lora = {}
    mods = dict(model.named_modules())
    for name in fo.lora_target_modules(cfg):
        lin = mods[name]
        lora[name] = ((torch.randn(32, lin.in_features, generator=g, device=dev) / lin.in_features ** 0.5).to(bf),
                      (torch.randn(lin.out_features, 32, generator=g, device=dev) * 0.09).to(bf))
    ls = fo.LoraSet(lora, 1.0)
    x = {k: (v.to(dev) if v is not None else None) for k, v in parity_inputs().items()}
    ts, sig = fo.flow_match_sigmas(max(steps, 1), N_IMG)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def run(n):
        lat = x["latents"]
        with torch.no_grad():
            for i in range(n):
                t = (ts[i].to(bf) / 1000).expand(1).to(dev)
                v = fo.transformer_forward(model, lat, x["prompt_embeds"], x["pooled"], t, x["img_ids"], x["txt_ids"],
                                           x["guidance"], x["cond_latents"], x["cond_ids"], {}, ls)
                lat = fo.euler_step(lat, v, sig[i], sig[i + 1])
        return lat
    run(2)
    torch.cuda.synchronize(dev)
    e0.record()
    run(steps)
    e1.record()
    torch.cuda.synchronize(dev)
    msps = e0.elapsed_time(e1) / steps
    tfl = algorithmic_tflop(N_TXT + N_IMG + N_COND, nl + ns)
    del model, lora
    torch.cuda.empty_cache()
    return {"value": 1e3 / msps, "unit": "denoise-steps/s", "ms_per_step": msps, "steps": steps,
            "tflops_achieved": tfl / (msps / 1e3),
            "how": "oracle/flux_oracle.py graph on cuda through stock torch ops (cuBLAS bf16 GEMMs, F.scaled_dot_product_attention, "
                   "eager elementwise), same 5632-token geometry incl. the peft-style unfused LoRA on every target (computed and "
                   "scaled by 0 on image tokens, as peft does), per-step RoPE / cond_temb recomputation as the reference does; "
                   "device-timed after 2 warm-up steps",
            "torch": torch.__version__}


if __name__ == "__main__":
    main()
