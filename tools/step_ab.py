#!/usr/bin/env python
"""dev tool: in-process A/B of launch-time switches on the denoise step (entry A 4608 tokens, entry B 5632 tokens
exact LoRA), alternated in ONE process so that box / clock state is shared.  Each argument is one variant: comma-
separated KEY=VALUE environment settings applied before its runs, which matter only for a switch the library reads at
graph-capture time.  The library reads none at present (RF_PDL is read once per process), so without arguments the
tool times the current build:  python tools/step_ab.py"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from reflectionflow_b200.pipeline import Condition, flow_match_schedule
from reflectionflow_b200.tts import reflectionflow as RF
from reflectionflow_b200.tts.dist import DistCtx

variants = [dict(kv.split("=") for kv in a.split(",")) for a in sys.argv[1:]] or [{}]
dev = torch.device("cuda:0")
ctx = DistCtx(0, 1, dev)
cfgj = json.load(open(os.path.join(os.path.dirname(RF.__file__), "configs", "headline_tree_flux_dev.json")))


class A:
    synthetic, layers, text_encoders, lora_mode = True, "19,38", "hash", "exact"


pipe = RF.build_pipeline(cfgj, A, ctx)
m = pipe.transformer
g = torch.Generator().manual_seed(0)
bf = torch.bfloat16
lat = torch.randn(1, 4096, 64, generator=g).to(bf).to(dev)
txt = torch.randn(1, 512, 4096, generator=g).to(bf).to(dev)
pool = torch.randn(1, 768, generator=g).to(bf).to(dev)
cond = torch.randn(1, 1024, 64, generator=g).to(bf).to(dev)
img_ids = pipe._prepare_latent_image_ids(1, 64, 64, dev, bf)
txt_ids = torch.zeros(512, 3, dtype=bf, device=dev)
_, cond_ids, _ = Condition("cot", latents=cond, position_delta=[0, -32]).encode(pipe)
K = int(os.environ.get("STEPS", "10"))
ts, sig = flow_match_schedule(K, 4096)
t_in = ts.to(bf) / 1000
lora = RF.synthetic_lora(m.cfg, seed=1)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def run(env, use_cond):
    os.environ.update(env)
    m.load_lora(lora, mode="exact")   # drops the captured graph: the next denoise re-captures under `env`
    a = (cond, cond_ids) if use_cond else (None, None)
    m.denoise(lat, txt, pool, t_in[:3], sig[:4], 3.5, img_ids, txt_ids, a[0], a[1], {})
    torch.cuda.synchronize()
    e0.record()
    m.denoise(lat, txt, pool, t_in, sig, 3.5, img_ids, txt_ids, a[0], a[1], {})
    e1.record()
    torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) / K, 2)


res = {json.dumps(v): {"entry_a": [], "entry_b": []} for v in variants}
for rep in range(3):
    for v in variants:
        res[json.dumps(v)]["entry_a"].append(run(v, False))
        res[json.dumps(v)]["entry_b"].append(run(v, True))
print(json.dumps(res))
