"""Time `B200FluxPipeline.from_pretrained` on a checkpoint directory and report its memory: wall time, peak host
RSS of this process, peak torch-allocated device memory (the staging copies) and device memory in use after the
load (the handles' weights).  One JSON line on stdout.

  python tools/measure_load.py CHECKPOINT_DIR [--lora-rank 32]

Files written just before are likely still in the page cache, so the time is then a cached read, not a disk read."""
from __future__ import annotations

import argparse
import json
import os
import resource
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("checkpoint")
    ap.add_argument("--lora-rank", type=int, default=0)
    a = ap.parse_args(argv)
    import torch
    from reflectionflow_b200.pipeline import B200FluxPipeline
    torch.cuda.init()
    free0, total = torch.cuda.mem_get_info()
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    pipe = B200FluxPipeline.from_pretrained(a.checkpoint, lora_rank=a.lora_rank)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    free1, _ = torch.cuda.mem_get_info()
    size = sum(os.path.getsize(os.path.join(d, f)) for d, _, fs in os.walk(a.checkpoint) for f in fs
               if f.endswith(".safetensors"))
    print(json.dumps({
        "gpu": torch.cuda.get_device_name(), "checkpoint_gb": round(size / 1e9, 2),
        "from_pretrained_s": round(wall, 2), "read_gb_per_s": round(size / 1e9 / wall, 2),
        "peak_host_rss_gb": round(resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20, 2),
        "host_rss_before_gb": round(rss0 / 2**20, 2),
        "peak_staging_gb": round(torch.cuda.max_memory_allocated() / 2**30, 3),
        "device_in_use_after_gb": round((free0 - free1) / 2**30, 2),
        "dit_layers": [pipe.transformer.cfg.num_layers, pipe.transformer.cfg.num_single_layers]}))


if __name__ == "__main__":
    main()
