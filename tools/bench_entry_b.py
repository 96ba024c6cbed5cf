#!/usr/bin/env python
"""Step time of entry B (condition stream + LoRA on condition tokens): the headline tree's step.

Env: LAYERS=double,single (default 19,38), LORA=0|1, LORA_MODE=exact|merged, LATENT_LORA=1 (the LoRA also acts on the
image and text tokens, model_config["latent_lora"]), LORA_RANK (default 32, up to 128), LORA_SCALE (default 1: the
call's joint_attention_kwargs["scale"]), LORA_TARGETS=config|all-linear (default config: the adapter covers the
Linears of train_flux/config.yaml:53; all-linear: every Linear of the transformer), IMAGE_GUIDANCE (default 1: generate's
image_guidance_scale; other values add the uncond forward to every step, with U_i = the condition latents), STEPS.
Prints the card name and power limit with the timing."""
import os, sys, json, subprocess, time
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from reflectionflow_b200 import _lib as L
from reflectionflow_b200.config import FluxDiTConfig
from reflectionflow_b200.pipeline import B200FluxPipeline, Condition, generate, flow_match_schedule
from reflectionflow_b200.tts.reflectionflow import synthetic_lora

dev = torch.device("cuda:0")
layers = os.environ.get("LAYERS", "19,38").split(",")
cfg = FluxDiTConfig(num_layers=int(layers[0]), num_single_layers=int(layers[1]))
use_lora = os.environ.get("LORA", "1") == "1"
latent_lora = os.environ.get("LATENT_LORA", "0") == "1"
lora_rank = int(os.environ.get("LORA_RANK", "32"))
lora_scale = float(os.environ.get("LORA_SCALE", "1"))
lora_targets = os.environ.get("LORA_TARGETS", "config")
image_guidance = float(os.environ.get("IMAGE_GUIDANCE", "1"))
model_config = {"union_cond_attn": True, "latent_lora": latent_lora}
jak = {"scale": lora_scale} if lora_scale != 1.0 else None
pipe = B200FluxPipeline.from_synthetic(cfg, seed=0, device=dev, lora_rank=lora_rank if use_lora else 0)
if use_lora:
    pipe.transformer.load_lora(synthetic_lora(cfg, rank=lora_rank, targets=lora_targets),
                               mode=os.environ.get("LORA_MODE", "exact"))
g = torch.Generator().manual_seed(0)
lat = torch.randn(1, 4096, 64, generator=g).to(torch.bfloat16)
txt = torch.randn(1, 512, 4096, generator=g).to(torch.bfloat16)
pool = torch.randn(1, 768, generator=g).to(torch.bfloat16)
cond = Condition("cot", latents=torch.randn(1, 1024, 64, generator=g).to(torch.bfloat16), position_delta=[0, -32])
K = int(os.environ.get("STEPS", "8"))
def run(n):
    return generate(pipe, conditions=[cond], model_config=model_config, default_lora=True, joint_attention_kwargs=jak,
                    image_guidance_scale=image_guidance,
                    prompt_embeds=txt, pooled_prompt_embeds=pool, latents=lat, height=1024, width=1024,
                    num_inference_steps=n, output_type="latent").images
run(3); torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); out = run(K); e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / K
tf = (57 * 24 * 3072 * 3072 * 5632 + 57 * 4 * 5632 * 5632 * 3072) / 1e12
try:
    power_limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                 capture_output=True, text=True, timeout=30).stdout.strip()
except Exception:
    power_limit = "unknown"
print(json.dumps({"entry": "B", "lora": use_lora, "lora_mode": pipe.transformer.lora_mode, "latent_lora": latent_lora,
                  "lora_rank": lora_rank if use_lora else 0, "lora_scale": lora_scale, "lora_targets": lora_targets,
                  "image_guidance_scale": image_guidance,
                  "n_tok": 5632, "ms_per_step": ms, "steps_per_s": 1e3 / ms, "step_tflop": tf, "tflops": tf / ms * 1e3,
                  "finite": bool(torch.isfinite(out.float()).all()), "gpu": torch.cuda.get_device_name(dev),
                  "power_limit": power_limit}))
from reflectionflow_b200.transformer import tranformer_forward
m = pipe.transformer
ids_i = pipe._prepare_latent_image_ids(1, 64, 64, dev, torch.bfloat16)
ids_t = torch.zeros(512, 3, dtype=torch.bfloat16, device=dev)
ctok, cids, _ = cond.encode(pipe)
kw = dict(hidden_states=lat, encoder_hidden_states=txt, pooled_projections=pool,
          timestep=torch.tensor([0.5], dtype=torch.bfloat16), img_ids=ids_i, txt_ids=ids_t,
          guidance=torch.tensor([3.5]), joint_attention_kwargs=jak, return_dict=False)
tranformer_forward(m, ctok, cids, None, model_config, 0, **kw)
torch.cuda.synchronize()
L.profile_start()
tranformer_forward(m, ctok, cids, None, model_config, 0, **kw)
prof = L.profile_stop()
tot = sum(v["ms"] for v in prof.values())
print(f"  one eager forward: {sum(v['launches'] for v in prof.values())} launches, {tot:.3f} ms of kernel time")
for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"]):
    print(f"  {k:20s} launches {v['launches']:4d}  ms {v['ms']:7.3f}  share {v['ms']/tot:.3f}")
