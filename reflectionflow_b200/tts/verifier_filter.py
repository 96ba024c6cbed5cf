"""Best-of-N filter over a finished run — mirror of tts/verifier_filter.py (main :28-176).  For every prompt
folder `NNNNN/{metadata.jsonl, midimg/<round>_round@<seed>.png}` written by the reflection loop, all candidates
are listed round by round (rounds in numeric order, files of a round in name order, :66-79), re-scored against the
prompt with the NVILA-shaped verifier (:107-113), and for N in 1, 2, 4, 8, 16, 32 the best of the FIRST N
candidates under the yes/no sort key (:119-123) is copied to `NNNNN/nfe<N>/00000.png` (:126-173).

Sharded form: scoring is sharded over the ranks and exchanged as fixed-size records (same helpers as the search
loops); every rank derives the same choices, rank 0 writes the files.  Candidates stored as `*.latent.pt`
(this framework always writes the packed latent next to the PNG) can be scored without a decode by verifiers
that do not need pixels, and are decoded through `pipe.vae` for the ones that do."""
from __future__ import annotations

import json
import os
import shutil
import time
from typing import Dict, List, Optional, Sequence

import torch

from . import search as S
from .dist import DistCtx
from .reflectionflow import _ensure_pixels, _exchange_outputs
from .utils import parse_cli_args
from .verifiers import Candidate, load_verifier

BUCKETS = (1, 2, 4, 8, 16, 32)


def list_candidates(folder: str) -> List[str]:
    """candidate stems `<folder>/midimg/<round>_round@<seed>` in the reference's order (:66-79)"""
    mid = os.path.join(folder, "midimg")
    by_round: Dict[str, List[str]] = {}
    seen = set()
    for fn in sorted(os.listdir(mid)):
        stem = fn[: -len(".latent.pt")] if fn.endswith(".latent.pt") else fn[:-4] if fn.endswith(".png") else None
        if stem is None or "_round@" not in stem or stem in seen:
            continue
        seen.add(stem)
        by_round.setdefault(stem.split("_round@")[0], []).append(stem)
    out = []
    for rk in sorted(by_round, key=int):
        out += [os.path.join(mid, s) for s in sorted(by_round[rk], key=lambda s: s + ".png")]
    return out


def load_candidate(stem: str, device="cpu") -> Candidate:
    seed = int(stem.split("@")[-1])
    lat = img = None
    if os.path.exists(stem + ".latent.pt"):
        lat = torch.load(stem + ".latent.pt", map_location="cpu").to(device)
    if os.path.exists(stem + ".png"):
        from PIL import Image
        with Image.open(stem + ".png") as im:
            img = im.convert("RGB").copy()
    return Candidate(stem + ".png", seed, latents=lat, image=img)


def best_of_first(outputs: Sequence[dict], n: int) -> int:
    """index (into outputs) of the best of the first n candidates under the NVILA key (:119-129)"""
    head = list(outputs[:n])
    return list(outputs).index(S.sort_outputs(head, "nvila")[0])


def filter_folder(folder: str, prompt: str, verifier, *, pipe=None, height: int = 1024, width: int = 1024,
                  ctx: Optional[DistCtx] = None, buckets: Sequence[int] = BUCKETS) -> dict:
    ctx = ctx or DistCtx()
    stems = list_candidates(folder)
    if not stems:
        raise RuntimeError(f"{folder}: no candidates under midimg/")
    cands = [load_candidate(s, ctx.device) for s in stems]
    mine = ctx.my_candidates(len(cands))
    t0 = time.time()
    if getattr(verifier, "needs_images", False):
        for i in mine:
            if cands[i].pil() is None:
                _ensure_pixels(pipe, cands[i], height, width)
                cands[i].pil()
    local_out = verifier.score([cands[i] for i in mine], [prompt] * len(mine))
    outputs = _exchange_outputs(ctx, "nvila", None, cands, mine, local_out)
    if ctx.rank == 0:
        print(f"Time taken for evaluation: {time.time() - t0} seconds")
    chosen = {}
    for n in buckets:
        k = best_of_first(outputs, n)
        chosen[n] = stems[k]
        if ctx.rank == 0:
            d = os.path.join(folder, f"nfe{n}")
            os.makedirs(d, exist_ok=True)
            for ext in (".png", ".latent.pt"):
                if os.path.exists(stems[k] + ext):
                    shutil.copyfile(stems[k] + ext, os.path.join(d, f"{0:05}" + ext))
    ctx.barrier()
    return {"outputs": outputs, "chosen": chosen}


@torch.no_grad()
def main(argv=None, ctx: Optional[DistCtx] = None):
    args = parse_cli_args(argv)
    with open(args.pipeline_config_path, "r") as f:
        config = json.load(f)
    config.update(vars(args))
    ctx = ctx or DistCtx.from_env()
    verifier_args = dict(config["verifier_args"], name="nvila")  # the reference filters with NVILA only (:47-48)
    verifier = load_verifier(verifier_args, args.synthetic)
    pipe = None
    if getattr(verifier, "needs_images", False):  # candidates stored as latents only need the VAE
        from .reflectionflow import build_pipeline
        pipe = build_pipeline(config, args, ctx)
    folders = [os.path.join(args.imgpath, d) for d in sorted(os.listdir(args.imgpath))
               if os.path.isdir(os.path.join(args.imgpath, d))]
    folders = folders[args.start_index:] if args.end_index == -1 else folders[args.start_index:args.end_index]
    pa = config["pipeline_args"]
    for folder in folders:
        with open(os.path.join(folder, "metadata.jsonl"), "r") as f:
            metadata = [json.loads(line) for line in f]
        filter_folder(folder, metadata[0]["prompt"], verifier, pipe=pipe, height=pa["height"], width=pa["width"],
                      ctx=ctx)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
