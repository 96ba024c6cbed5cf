"""Noise + prompt-refinement search — mirror of tts/tts_t2i_noise_prompt_scaling.py (sample :22-145,
main :149-248).  Per prompt x round: draw `search_branch` seeded noises (`get_noises`), generate one
image per (noise, current prompt) with the stock FLUX pipeline (entry A, `pipe(prompt=, latents=, ...)`,
:79), score every image against the ORIGINAL prompt (:98-121, the sort keys of `search.sort_outputs`),
take the top-k indices (:123-124), then let the refiner rewrite every current prompt from (image,
evaluation, original prompt, current prompt) for the next round (:127-137); `refined_prompt<r>` is appended
to `best_img_meta.jsonl` (:139-140).

Sharded form: the candidates of a round are sharded over the ranks (one process per GPU), final latents and
score records are all-gathered (as in `reflectionflow.sample`), every rank derives the same ranking, the LLM
hook runs on rank 0 and its text is broadcast.  The verifier / refiner networks are external models behind
`verifiers.load_verifier` / the reflector classes (stubs offline)."""
from __future__ import annotations

import copy
import json
import os
import time
from typing import Callable, Dict, List, Optional, Union

import torch

from . import search as S
from .dist import DistCtx
from .reflectionflow import (_ensure_pixels, _exchange_outputs, _rank0_call, _save_candidate, build_pipeline,
                             flush_saves)
from .utils import TORCH_DTYPE_MAP, get_latent_prep_fn, get_noises, parse_cli_args
from .verifiers import Candidate, StubReflector, StubVerifier, load_verifier

MAX_SEED = S.MAX_SEED


def sample(noises: Dict[int, torch.Tensor], original_prompt: str, updated_prompt: Union[str, List[str]],
           search_round: int, pipe, topk: int, root_dir: str, config: dict, midimg_path: str,
           tag: Optional[str] = None, *, verifier=None, refiner=None, ctx: Optional[DistCtx] = None,
           pixels_fn: Callable = _ensure_pixels, defer_saves: bool = False) -> dict:
    """One round.  Returns the reference's datapoint (`original_prompt`, `refined_prompt`, `search_round`,
    `num_noises`, `choice_of_metric`) plus what the sharded loop needs (`topk_idx`, `scores`, `generated`)."""
    ctx = ctx or DistCtx()
    config_cp = copy.deepcopy(config)
    verifier_name = config["verifier_args"].get("name", "openai")
    refine_args = config["refine_args"]
    choice_of_metric = refine_args.get("choice_of_metric", None)
    verifier = verifier or StubVerifier(verifier_name, choice_of_metric or "overall_score")
    refiner = refiner or StubReflector()
    bs = config_cp.get("batch_size_for_img_gen", 1)
    pa = config_cp["pipeline_args"]
    rank0 = ctx.rank == 0
    num = len(noises)
    prompts = list(updated_prompt) if isinstance(updated_prompt, (list, tuple)) else [updated_prompt] * num
    if len(prompts) != num:
        raise ValueError(f"{len(prompts)} prompts for {num} noises")

    # ---- generate: my share of the (noise, prompt) pairs, in batches (:62-88)
    noise_items = list(noises.items())
    names = [os.path.join(midimg_path, f"{search_round}_round@{seed}.png") for seed, _ in noise_items]
    mine = ctx.my_candidates(num)
    local = []
    for b0 in range(0, len(mine), bs):
        idxs = mine[b0:b0 + bs]
        if rank0:
            print(f"Generating images for batch with seeds: {[noise_items[i][0] for i in idxs]}.")
        batched_latents = torch.stack([noise_items[i][1] for i in idxs]).squeeze(dim=1)
        res = pipe(prompt=[prompts[i] for i in idxs], latents=batched_latents,
                   guidance_scale=pa["guidance_scale"], num_inference_steps=pa["num_inference_steps"],
                   height=pa["height"], width=pa["width"], output_type="latent")
        for j, i in enumerate(idxs):
            local.append((i, res.images[j:j + 1]))

    # ---- exchange the final latents (the refiner on rank 0 looks at every image), decode / store my own
    shape = tuple(local[0][1].shape) if local else tuple(noise_items[0][1].shape)
    shape = tuple(ctx.broadcast_object(shape))
    all_lat = ctx.gather_latents(local, num, shape, torch.bfloat16)
    cands = [Candidate(names[i], noise_items[i][0], latents=all_lat[i]) for i in range(num)]
    for i in mine:
        pixels_fn(pipe, cands[i], pa["height"], pa["width"])
        _save_candidate(cands[i], names[i])

    # ---- score against the original prompt (sharded), exchange, rank (:92-124)
    t0 = time.time()
    if getattr(verifier, "needs_images", False):
        for i in mine:
            cands[i].pil()
    local_out = verifier.score([cands[i] for i in mine], [original_prompt] * len(mine), tag=tag)
    outputs = _exchange_outputs(ctx, verifier_name, choice_of_metric, cands, mine, local_out)
    sorted_list = S.sort_outputs(outputs, verifier_name, choice_of_metric)
    if rank0:
        print(f"Time taken for evaluation: {time.time() - t0} seconds")
    topk_idx, _selected, _sel_out = S.select_topk(outputs, sorted_list, cands, topk)

    # ---- refine every prompt for the next round (:127-137): rank 0 asks, everybody gets the text
    evaluations = [json.dumps(o) for o in outputs]
    wants_pixels = getattr(refiner, "needs_images", not isinstance(refiner, StubReflector))

    def refine():
        if wants_pixels:
            for c in cands:
                pixels_fn(pipe, c, pa["height"], pa["width"])
                c.pil()
        return refiner.refine_prompt(cands, original_prompt, prompts, None,
                                     evaluations if verifier_name == "openai" else None)

    refined = list(_rank0_call(ctx, refine))
    if len(refined) != len(prompts):  # the reference asserts the same (:136)
        raise RuntimeError(f"refiner returned {len(refined)} prompts for {len(prompts)}")
    if rank0:
        with open(os.path.join(root_dir, "best_img_meta.jsonl"), "a") as f:
            f.write(f"refined_prompt{search_round}: " + json.dumps(refined) + "\n")
    if not defer_saves:
        flush_saves()
        ctx.barrier()
    return {"original_prompt": original_prompt, "refined_prompt": refined, "search_round": search_round,
            "num_noises": num, "choice_of_metric": choice_of_metric,
            "topk_idx": topk_idx, "scores": outputs, "generated": cands}


@torch.no_grad()
def main(argv=None, ctx: Optional[DistCtx] = None, *, verifier=None, refiner=None):
    """tts_t2i_noise_prompt_scaling.py:149-248 (output layout NNNNN/{metadata.jsonl, samples/, best_img_meta.jsonl}).
    `verifier` / `refiner` inject the external models (default: the config's verifier, the offline stub refiner)."""
    args = parse_cli_args(argv)
    with open(args.pipeline_config_path, "r") as f:
        config = json.load(f)
    config.update(vars(args))
    config.setdefault("use_low_gpu_vram", False)
    ctx = ctx or DistCtx.from_env()
    if args.seed is not None:
        torch.manual_seed(args.seed)
    else:  # the reference is unseeded; ranks must still agree on the seed stream
        torch.manual_seed(int(ctx.broadcast_object(int(torch.seed() % (2 ** 31)))))
    search_rounds = config["search_args"]["search_rounds"]
    search_branch = config["search_args"]["search_branch"]
    pipeline_name = config["pipeline_args"].get("pretrained_model_name_or_path")
    root_dir = config["output_dir"]
    os.makedirs(root_dir, exist_ok=True)
    torch_dtype = TORCH_DTYPE_MAP[config["pipeline_args"].get("torch_dtype")]
    cfg_noload = dict(config)
    cfg_noload["pipeline_args"] = dict(config["pipeline_args"], lora_path=None)  # entry A: no LoRA
    pipe = build_pipeline(cfg_noload, args, ctx)
    verifier = verifier or load_verifier(config["verifier_args"], args.synthetic,
                                         config["refine_args"].get("choice_of_metric", "overall_score"))
    refiner = refiner or StubReflector()  # an OpenAIShapedReflector(client, ...) when a client is available
    with open(args.meta_path) as fp:
        metadatas = [json.loads(line) for line in fp]
    metadatas = metadatas[args.start_index:] if args.end_index == -1 else \
        metadatas[args.start_index:args.end_index]
    for index, metadata in enumerate(metadatas):
        outpath = os.path.join(root_dir, f"{index + args.start_index:0>5}")
        midimg_path = os.path.join(outpath, "samples")
        if ctx.rank == 0:
            os.makedirs(midimg_path, exist_ok=True)
            with open(os.path.join(outpath, "metadata.jsonl"), "w") as fp:
                json.dump(metadata, fp)
        ctx.barrier()
        original_prompt = metadata["prompt"]
        updated_prompt = [original_prompt] * search_branch
        for rnd in range(1, search_rounds + 1):
            if ctx.rank == 0:
                print(f"\n=== Round: {rnd} ===")
            noises = get_noises(max_seed=MAX_SEED, num_samples=search_branch,
                                height=config["pipeline_args"]["height"],
                                width=config["pipeline_args"]["width"], dtype=torch_dtype,
                                fn=get_latent_prep_fn(pipeline_name))
            if ctx.rank == 0:
                print(f"Number of noise samples: {len(noises)}")
            dp = sample(noises=noises, original_prompt=original_prompt, updated_prompt=updated_prompt,
                        search_round=rnd, pipe=pipe, topk=search_branch, root_dir=outpath, config=config,
                        midimg_path=midimg_path, tag=metadata.get("tag"), verifier=verifier, refiner=refiner,
                        ctx=ctx, defer_saves=True)
            updated_prompt = dp["refined_prompt"]
    flush_saves()
    ctx.barrier()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
