"""ReflectionFlow search loop on sharded GPUs — mirror of tts/tts_reflectionflow.py (sample :94-463,
main :466-629): per round  score parents -> top-k -> reflect -> refine prompt -> regenerate each
candidate conditioned on its parent -> re-score -> chain bookkeeping.

What changes, and why (SURVEY.md §8e, App. B):
  * candidates of a round are sharded over the ranks (candidate i -> rank i mod world); each rank
    runs full denoise trajectories on its own GPU; ONE all-gather of score records (+ one of the
    candidates' packed latents, the next round's parents) per round; every rank then runs the same
    deterministic selection, so all ranks agree on top-k indices bit for bit;
  * the boundary is explicit: init noise = the `noises` the caller sampled (the reference samples
    them but never passes them on, App. B.1), condition latents are given tensors (the reference
    samples the VAE posterior, B.4);
  * images cross rounds in HBM, not as PNG files re-opened from disk: with a VAE attached the
    parent -> condition step is decode -> PIL-exact BICUBIC resize -> encode, all on the device
    (PNGs are still written for downstream tools); a pipeline without a VAE cannot form the
    condition and raises.
Artefact layout and names (midimg/<round>_round@<seed>.png, best_img_meta.jsonl,
best_img_detailedscore.jsonl, samples_best/, samples_lastround/, samples_path_bestround/) follow the
reference so downstream tools keep working."""
from __future__ import annotations

import copy
import json
import os
import time
from typing import Callable, Dict, List, Optional, Union

import torch

from ..pipeline import Condition, generate as _generate
from . import search as S
from .dist import DistCtx
from .utils import TORCH_DTYPE_MAP, get_latent_prep_fn, get_noises, parse_cli_args
from .verifiers import Candidate, HashTextEncoder, StubReflector, StubVerifier, load_verifier

MAX_SEED = S.MAX_SEED
MAX_RETRIES = 5
RETRY_DELAY = 2


_SAVER = None
_PENDING: Dict[str, "object"] = {}
# every candidate of the current prompt's tree by name (the reference re-opens PNGs from disk when it
# copies a best image of an EARLIER round, tts_reflectionflow.py:408-446; a tree is 32 candidates of
# 0.5 MB latents + 3 MB pixels, so they simply stay referenced until the next prompt)
_REGISTRY: Dict[str, Dict[str, Candidate]] = {}


def _registry(root_dir: str, search_round: int) -> Dict[str, Candidate]:
    if search_round == 1:
        _REGISTRY.clear()  # one prompt's tree at a time
    return _REGISTRY.setdefault(root_dir, {})



def _submit_save(path: str, job: Callable[[], None]):
    """Artefact writes run on a small thread pool (PNG deflate releases the GIL) so that they overlap
    the next candidate's denoise instead of sitting on the critical path; writes to the same path keep
    their order.  `flush_saves()` joins them."""
    global _SAVER
    if _SAVER is None:
        from concurrent.futures import ThreadPoolExecutor
        _SAVER = ThreadPoolExecutor(max_workers=int(os.environ.get("RF_SAVE_THREADS", "8")))
    prev = _PENDING.get(path)

    def run():
        if prev is not None:
            prev.result()  # submitted earlier, hence already running or done: cannot deadlock
        job()
    _PENDING[path] = _SAVER.submit(run)


def flush_saves():
    """Block until every artefact submitted so far is on disk (re-raises a failed write)."""
    pending = list(_PENDING.items())
    _PENDING.clear()
    for _path, fut in pending:
        fut.result()


def _save_candidate(cand: Candidate, path: str):
    """PNG when the candidate has pixels (VAE attached), always the packed latent next to it (the
    next stage reloads candidates from `*.latent.pt`, not by re-encoding PNGs).  Device->host copies
    happen here, on the calling thread; encoding and file IO on the save workers."""
    if cand.pil() is not None:
        def write_png(c=cand, p=path):
            with open(p, "wb") as f:
                f.write(c.png_bytes())
        _submit_save(path, write_png)
    if cand.latents is not None:
        lat, lp = cand.latents.cpu(), os.path.splitext(path)[0] + ".latent.pt"
        _submit_save(lp, lambda: torch.save(lat, lp))


def _ensure_pixels(pipe, cand: Candidate, height: int, width: int):
    if cand.image_u8 is None and getattr(pipe, "vae", None) is not None:
        cand.image_u8 = pipe.vae.decode_packed(cand.latents.reshape(1, -1, cand.latents.shape[-1]),
                                               height, width, "u8")[0]
    return cand.image_u8


def parent_condition(pipe, parent: Candidate, height: int, width: int, cond_size: int, seed: int):
    """tts_reflectionflow.py:273-279: the parent IMAGE, resized to condition_size, becomes the `cot`
    condition.  With a VAE attached this is the real path, all on the device: decode -> PIL-exact
    BICUBIC resize -> encode (posterior noise seeded by the candidate's seed).  There is no
    latent-space stand-in: without a VAE the condition cannot be formed."""
    position_delta = [0, -cond_size // 16]
    if getattr(pipe, "vae", None) is None:
        raise RuntimeError("the reflection loop needs pipe.vae (decode -> resize -> encode of the parent "
                           "image, tts_reflectionflow.py:273-279); build the pipeline with with_vae=True")
    from ..resize import resize_u8
    u8 = _ensure_pixels(pipe, parent, height, width)
    small = resize_u8(u8[None], cond_size, cond_size)
    eps = torch.randn((16, cond_size // 8, cond_size // 8), generator=torch.Generator().manual_seed(int(seed)),
                      dtype=torch.bfloat16)
    return Condition("cot", condition=small, position_delta=position_delta, eps=eps)


def sample(noises: Dict[int, torch.Tensor], original_prompt: str,
           updated_prompt: Union[str, List[str]], reflections: Union[str, List[str]],
           search_round: int, pipe, topk: int, root_dir: str, config: dict,
           sample_path_lastround: str, sample_path_best: str, sample_path_bestround: str,
           imagetoupdate: List[Candidate], midimg_path: str, total_rounds: int, chains: dict,
           tag: Optional[str] = None, *, verifier=None, reflector=None, ctx: Optional[DistCtx] = None,
           generate_fn: Callable = _generate, defer_saves: bool = False,
           condition_fn: Optional[Callable] = None) -> dict:
    """`defer_saves=True` leaves artefact writes in flight when the round returns (they overlap the
    next round; the caller ends with `flush_saves()`); by default the round's files are on disk."""
    ctx = ctx or DistCtx()
    verifier = verifier or StubVerifier(config["verifier_args"].get("name", "openai"))
    reflector = reflector or StubReflector()
    flag_terminated = search_round == total_rounds
    config_cp = copy.deepcopy(config)
    verifier_name = config["verifier_args"].get("name", "openai")
    refine_args = config["refine_args"]
    choice_of_metric = refine_args.get("choice_of_metric", None)
    reflection_args = config_cp.get("reflection_args", None)
    num_samples = len(noises)
    rank0 = ctx.rank == 0
    pa = config_cp["pipeline_args"]

    # ---- 1. score the parents (sharded) and exchange the records
    t0 = time.time()
    n_prev = len(imagetoupdate)
    mine = ctx.my_candidates(n_prev)
    if getattr(verifier, "needs_images", False):  # real verifiers look at pixels: decode the parents
        for i in mine:
            _ensure_pixels(pipe, imagetoupdate[i], pa["height"], pa["width"])
            imagetoupdate[i].pil()
    local_out = verifier.score([imagetoupdate[i] for i in mine], [original_prompt] * len(mine), tag=tag)
    outputs = _exchange_outputs(ctx, verifier_name, choice_of_metric, imagetoupdate, mine, local_out)
    sorted_list = S.sort_outputs(outputs, verifier_name, choice_of_metric)
    if rank0:
        print(f"Time taken for evaluation: {time.time() - t0} seconds")

    # ---- 2. top-k (identical on every rank)
    topk_idx, selected, selected_outputs = S.select_topk(outputs, sorted_list, imagetoupdate, topk)
    selected_imgs = [c.name for c in selected]
    if rank0:
        with open(os.path.join(root_dir, "best_img_detailedscore.jsonl"), "a") as f:
            f.write(json.dumps({"evaluation": selected_outputs, "filenames_batch": selected_imgs}) + "\n")

    # ---- 3./4. reflections and prompt refinement: rank 0 asks the LLM hooks, everybody gets the text
    reflection_performed = refinement_performed = False
    update_reflections, refined_prompt = None, None
    evaluations = [json.dumps(o) for o in selected_outputs]
    # LLM hooks that look at the images (everything but the stub) need the selected parents' pixels on rank 0,
    # whichever rank generated them and whether or not the verifier needed pixels
    wants_pixels = getattr(reflector, "needs_images", not isinstance(reflector, StubReflector))

    def hook_pixels():
        if wants_pixels:
            for c in selected:
                _ensure_pixels(pipe, c, pa["height"], pa["width"])
                c.pil()
    if reflection_args and reflection_args.get("run_reflection", False):
        t0 = time.time()
        def reflect():
            retries = 0
            hook_pixels()
            while True:
                try:
                    return reflector.generate_reflections(
                        selected, original_prompt, updated_prompt, reflections, evaluations)
                except Exception as e:  # tts_reflectionflow.py:208-219
                    retries += 1
                    if retries >= MAX_RETRIES:
                        raise
                    print(f"Error generating reflection: {e}. Retrying in {RETRY_DELAY} seconds...")
                    time.sleep(RETRY_DELAY)
        update_reflections = _rank0_call(ctx, reflect)
        reflection_performed = True
        if rank0:
            print(f"Time taken for reflection generation: {time.time() - t0} seconds")
    prompt_refiner_args = config_cp.get("prompt_refiner_args", None)
    if prompt_refiner_args and prompt_refiner_args.get("run_refinement", False):
        t0 = time.time()
        def refine():
            hook_pixels()
            return reflector.refine_prompt(selected, original_prompt, updated_prompt, update_reflections,
                                           evaluations if verifier_name == "openai" else None)
        refined_prompt = _rank0_call(ctx, refine)
        refinement_performed = True
        if rank0:
            print(f"Time taken for prompt refinement: {time.time() - t0} seconds")
    if rank0 and (reflection_performed or refinement_performed):
        with open(os.path.join(root_dir, "best_img_meta.jsonl"), "a") as f:
            if reflection_performed:
                f.write(f"reflections{search_round}: " + json.dumps(update_reflections) + "\n")
            if refinement_performed:
                f.write(f"refined_prompt{search_round}: " + json.dumps(refined_prompt) + "\n")
            f.write(f"filenames_batch{search_round}: " + json.dumps(selected_imgs) + "\n")

    # ---- 5./6. prompts and conditions (tts_reflectionflow.py:273-294)
    if reflection_args and reflection_args.get("run_reflection", False):
        base = refined_prompt if refined_prompt is not None else updated_prompt
        prompts = S.compose_prompts(base, update_reflections)
    else:
        prompts = [original_prompt] * num_samples
    cond_size = pa["condition_size"]

    # ---- 7. regenerate: my share of the candidates, one full trajectory each
    t0 = time.time()
    noise_items = list(noises.items())
    full_imgnames = [os.path.join(midimg_path, f"{search_round}_round@{seed}.png") for seed, _ in noise_items]
    new_local = []
    for i in ctx.my_candidates(num_samples):
        seed, noise = noise_items[i]
        parent = selected[i]
        cond = (condition_fn or parent_condition)(pipe, parent, pa["height"], pa["width"], cond_size, seed)
        result = generate_fn(pipe, prompt=[prompts[i]], conditions=[cond], height=pa["height"],
                             width=pa["width"], model_config=config.get("model", None),
                             default_lora=True, latents=noise, output_type="latent")
        new_local.append((i, Candidate(full_imgnames[i], seed, latents=result.images)))
    if rank0:
        print(f"Time taken for image generation: {time.time() - t0} seconds")

    # ---- 8. exchange: latents of all new candidates (next round's parents), then their scores
    shape = tuple(new_local[0][1].latents.shape) if new_local else tuple(noise_items[0][1].shape)
    shape = tuple(ctx.broadcast_object(shape))
    all_lat = ctx.gather_latents([(i, c.latents) for i, c in new_local], num_samples, shape,
                                 torch.bfloat16)
    new_cands = [Candidate(full_imgnames[i], noise_items[i][0], latents=all_lat[i])
                 for i in range(num_samples)]
    for i, _c in new_local:  # each rank decodes (VAE attached) and stores its own candidates
        _ensure_pixels(pipe, new_cands[i], pa["height"], pa["width"])
        _save_candidate(new_cands[i], full_imgnames[i])
    t0 = time.time()
    mine = ctx.my_candidates(num_samples)
    if getattr(verifier, "needs_images", False):
        for i in mine:
            new_cands[i].pil()
    local_out = verifier.score([new_cands[i] for i in mine], [original_prompt] * len(mine), tag=tag)
    outputs = _exchange_outputs(ctx, verifier_name, choice_of_metric, new_cands, mine, local_out)
    if rank0:
        print(f"Time taken for evaluation: {time.time() - t0} seconds")

    # ---- 9. chains / best-of bookkeeping (identical on every rank; files from rank 0)
    S.update_chains(chains, search_round, full_imgnames, outputs, selected_imgs, verifier_name,
                    choice_of_metric)
    by_name = _registry(root_dir, search_round)
    for c in list(imagetoupdate) + new_cands:
        by_name[c.name] = c

    def materialise(name: str) -> Candidate:
        if name not in by_name:
            raise RuntimeError(f"best candidate {name} of an earlier round is not in the registry")
        c = by_name[name]
        _ensure_pixels(pipe, c, pa["height"], pa["width"])
        return c
    if rank0:
        if search_round == total_rounds:
            for i, c in enumerate(new_cands):
                _save_candidate(c, os.path.join(sample_path_lastround, f"{i:05}.png"))
        if search_round == 1:
            for i, c in enumerate(new_cands):
                _save_candidate(c, os.path.join(sample_path_bestround, f"{i:05}.png"))
        else:
            for i, name in enumerate(S.best_per_chain(chains, verifier_name)):
                _save_candidate(materialise(name), os.path.join(sample_path_bestround, f"{i:05}.png"))
        if search_round == total_rounds:
            best = S.global_best(chains, verifier_name)
            # the reference names this file with a leaked loop index (App. B.9); we use 00000
            _save_candidate(materialise(best), os.path.join(sample_path_best, f"{0:05}.png"))

    datapoint = {"original_prompt": original_prompt, "search_round": search_round,
                 "num_noises": len(noises), "choice_of_metric": choice_of_metric,
                 "generated_img": full_imgnames, "generated": new_cands,
                 "flag_terminated": flag_terminated, "chains": chains, "topk_idx": topk_idx,
                 "scores": outputs}
    if refinement_performed:
        datapoint["refined_prompt"] = refined_prompt
    if reflection_performed:
        datapoint["reflections"] = update_reflections
    if not defer_saves:
        flush_saves()
    return datapoint


def _rank0_call(ctx: DistCtx, fn: Callable):
    """Run an LLM hook on rank 0 and give every rank its result; a failure on rank 0 is broadcast
    too, so all ranks raise together instead of hanging in the collective."""
    box = None
    if ctx.rank == 0:
        try:
            box = ("ok", fn())
        except Exception as e:  # noqa: BLE001 - re-raised on every rank below
            box = ("err", f"{type(e).__name__}: {e}")
    box = ctx.broadcast_object(box)
    if box[0] == "err":
        raise RuntimeError(f"rank-0 hook failed: {box[1]}")
    return box[1]


def _exchange_outputs(ctx: DistCtx, verifier_name: str, metric: str, cands: List[Candidate],
                      mine: List[int], local_out: List[dict]) -> List[dict]:
    """All-gather fixed-size (cand_id, seed, label, score) records — the selection key, identical
    on every rank — and rebuild the reference-shaped output dicts in candidate order.  The nvila
    dict is exactly its record; richer verifier outputs (every aspect + explanation of the
    OpenAI-shaped JSON, which feeds generate_reflections / refine_prompt and
    best_img_detailedscore.jsonl, tts_reflectionflow.py:184-257) travel whole, as objects."""
    recs = []
    for i, o in zip(mine, local_out):
        if verifier_name == "nvila":
            recs.append((i, cands[i].seed, 1 if o["label"] == "yes" else 0, float(o["score"])))
        else:
            recs.append((i, cands[i].seed, 1, float(S.metric_value(o, metric))))
    allr = ctx.gather_records(recs, len(cands))
    full = {}
    if verifier_name != "nvila":
        for part in ctx.gather_objects([(i, o) for i, o in zip(mine, local_out)]):
            full.update(dict(part))
    outs = []
    for cid, seed, label, score in allr:
        if verifier_name == "nvila":
            outs.append({"image_name": cands[cid].name, "label": "yes" if label else "no", "score": score})
        else:
            o = dict(full[cid])  # as the verifier returned it (the reference adds nothing, :146-151)
            if float(S.metric_value(o, metric)) != float(score):
                raise RuntimeError(f"candidate {cid}: score record and verifier output disagree")
            outs.append(o)
    return outs


def build_pipeline(config: dict, args, ctx: DistCtx):
    """DiffusionPipeline.from_pretrained(...).to("cuda") + load_lora_weights
    (tts_reflectionflow.py:498-505): the checkpoint `pretrained_model_name_or_path` names (a directory, or a
    repo id in the hub cache under `cache_dir`), read from disk by every rank onto its own device, with the
    adapter at `lora_path` (its rank sizes the transformer's LoRA slots).  Offline (--synthetic): random-init
    weights of the FLUX.1-dev architecture, seeded identically on every rank, random LoRA, hash text
    embeddings."""
    from ..config import FluxDiTConfig
    from ..pipeline import B200FluxPipeline
    pa = config["pipeline_args"]
    cfg = FluxDiTConfig()
    if getattr(args, "layers", None):
        nl, ns = (int(v) for v in args.layers.split(","))
        cfg = FluxDiTConfig(num_layers=nl, num_single_layers=ns)
    lora_path = pa.get("lora_path", None)
    if not getattr(args, "synthetic", False):
        from ..checkpoint import max_lora_rank
        pipe = B200FluxPipeline.from_pretrained(
            pa["pretrained_model_name_or_path"], cache_dir=pa.get("cache_dir"), torch_dtype=pa.get("torch_dtype"),
            device=ctx.device, lora_rank=max_lora_rank(lora_path) if lora_path is not None else 0)
        if lora_path is not None:
            pipe.transformer.lora_mode = getattr(args, "lora_mode", None) or "exact"
            pipe.load_lora_weights(lora_path, adapter_name="reflection")
        pipe.set_progress_bar_config(disable=True)
        return pipe
    pipe = B200FluxPipeline.from_synthetic(cfg, seed=0, device=ctx.device,
                                           lora_rank=32 if lora_path is not None else 0, with_vae=True)
    if getattr(args, "text_encoders", "hash") == "native":
        # T5-v1.1-XXL + CLIP-L of the real shapes (random init), ids from a byte tokenizer stand-in
        from ..text import B200TextEncoders
        from .verifiers import ByteTokenizer
        enc = B200TextEncoders(device=ctx.device).init_synthetic_weights(seed=2)
        pipe.text_encoders = enc
        pipe.text_encoder_hook = enc.as_hook(ByteTokenizer(49408, eos=49407, pad=49407, bos=49406),
                                             ByteTokenizer(32128, eos=1, pad=0))
    else:
        pipe.text_encoder_hook = HashTextEncoder(cfg.joint_attention_dim, cfg.pooled_projection_dim)
    if lora_path is not None:
        # "exact" = peft's unfused arithmetic (what the reference runs); "merged" = fuse_lora
        pipe.transformer.load_lora(synthetic_lora(cfg, seed=1), mode=getattr(args, "lora_mode", None) or "exact")
    pipe.set_progress_bar_config(disable=True)
    return pipe


def synthetic_lora(cfg, rank: int = 32, seed: int = 1, targets: str = "config"):
    """Random LoRA factors on the target list of train_flux/config.yaml:53 (targets="config"), or on every Linear of
    the transformer (targets="all-linear", train/model.py:73-80).  The config.yaml:53 factors are the same either
    way: the other Linears draw afterwards from the same generator."""
    if targets not in ("config", "all-linear"):
        raise ValueError(f"targets must be 'config' or 'all-linear', got {targets!r}")
    d = cfg.inner_dim
    g = torch.Generator().manual_seed(seed)
    out = {}

    def add(name, o, i):
        out[name] = ((torch.randn(rank, i, generator=g) / i ** 0.5).to(torch.bfloat16),
                     (torch.randn(o, rank, generator=g) * (0.5 / rank ** 0.5)).to(torch.bfloat16))
    add("x_embedder", d, cfg.in_channels)
    for i in range(cfg.num_layers):
        p = f"transformer_blocks.{i}."
        add(p + "norm1.linear", 6 * d, d)
        for n in ("attn.to_q", "attn.to_k", "attn.to_v", "attn.to_out.0"):
            add(p + n, d, d)
        add(p + "ff.net.2", d, 4 * d)
    for i in range(cfg.num_single_layers):
        p = f"single_transformer_blocks.{i}."
        add(p + "norm.linear", 3 * d, d)
        add(p + "proj_mlp", 4 * d, d)
        add(p + "proj_out", d, 5 * d)
        for n in ("attn.to_q", "attn.to_k", "attn.to_v"):
            add(p + n, d, d)
    if targets == "all-linear":
        add("context_embedder", d, cfg.joint_attention_dim)
        tte = "time_text_embed."
        add(tte + "timestep_embedder.linear_1", d, 256)
        add(tte + "timestep_embedder.linear_2", d, d)
        if cfg.guidance_embeds:
            add(tte + "guidance_embedder.linear_1", d, 256)
            add(tte + "guidance_embedder.linear_2", d, d)
        add(tte + "text_embedder.linear_1", d, cfg.pooled_projection_dim)
        add(tte + "text_embedder.linear_2", d, d)
        for i in range(cfg.num_layers):
            p = f"transformer_blocks.{i}."
            add(p + "norm1_context.linear", 6 * d, d)
            for n in ("attn.add_q_proj", "attn.add_k_proj", "attn.add_v_proj", "attn.to_add_out"):
                add(p + n, d, d)
            add(p + "ff.net.0.proj", 4 * d, d)
            add(p + "ff_context.net.0.proj", 4 * d, d)
            add(p + "ff_context.net.2", d, 4 * d)
        add("norm_out.linear", 2 * d, d)
        add("proj_out", cfg.in_channels, d)
    return out


@torch.no_grad()
def main(argv=None, ctx: Optional[DistCtx] = None, *, verifier=None, reflector=None,
         generate_fn: Optional[Callable] = None, condition_fn: Optional[Callable] = None):
    """tts_reflectionflow.py:466-629.  `--imgpath` holds the round-0 candidates written by the
    noise-scaling stage (NNNNN/{metadata.jsonl, samples/*}); each rank owns a share of every round.
    `verifier` / `reflector` inject the external models (default: what the config names, stubs with --synthetic);
    `generate_fn` / `condition_fn` replace the denoiser and the parent -> condition step (tests)."""
    args = parse_cli_args(argv)
    with open(args.pipeline_config_path, "r") as f:
        config = json.load(f)
    config.update(vars(args))
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
    pipe = build_pipeline(config, args, ctx)
    verifier_args = config["verifier_args"]
    verifier_name = verifier_args.get("name", "openai")
    verifier = verifier or load_verifier(verifier_args, args.synthetic,
                                         config["refine_args"].get("choice_of_metric", "overall_score"))
    reflector = reflector or StubReflector()
    hooks = {}
    if generate_fn is not None:
        hooks["generate_fn"] = generate_fn
    if condition_fn is not None:
        hooks["condition_fn"] = condition_fn
    use_reflection = (config.get("reflection_args") or {}).get("run_reflection", False)
    use_refine = (config.get("prompt_refiner_args") or {}).get("run_refinement", False)

    metadatas = []
    for folder_name in sorted(os.listdir(args.imgpath)):
        folder_path = os.path.join(args.imgpath, folder_name)
        if not os.path.isdir(folder_path):
            continue
        with open(os.path.join(folder_path, "metadata.jsonl"), "r") as f:
            metadata = [json.loads(line) for line in f]
        samples_path = os.path.join(folder_path, "samples")
        images = []
        if os.path.exists(samples_path):
            images = [os.path.join(samples_path, fn) for fn in sorted(os.listdir(samples_path))]
        metadatas.append({"metadata": metadata, "images": images})
    metadatas = metadatas[args.start_index:] if args.end_index == -1 else \
        metadatas[args.start_index:args.end_index]

    for index, metadata in enumerate(metadatas):
        meta0 = metadata["metadata"][0]
        outpath = os.path.join(root_dir, f"{index + args.start_index:0>5}")
        dirs = {k: os.path.join(outpath, k) for k in
                ("samples_lastround", "samples_best", "samples_path_bestround", "midimg")}
        if ctx.rank == 0:
            for d in dirs.values():
                os.makedirs(d, exist_ok=True)
            with open(os.path.join(outpath, "metadata.jsonl"), "w") as fp:
                json.dump(meta0, fp)
        ctx.barrier()
        updated_prompt = [meta0["prompt"]] * search_branch
        original_prompt = meta0["prompt"]
        reflections = [""] * search_branch if use_reflection else None
        imagetoupdate = load_round0(metadata["images"], ctx)
        chains = {}
        for rnd in range(1, search_rounds + 1):
            if ctx.rank == 0:
                print(f"\n=== Round: {rnd} ===")
            noises = get_noises(max_seed=MAX_SEED, num_samples=search_branch,
                                height=config["pipeline_args"]["height"],
                                width=config["pipeline_args"]["width"], dtype=torch_dtype,
                                fn=get_latent_prep_fn(pipeline_name))
            dp = sample(noises=noises, original_prompt=original_prompt, updated_prompt=updated_prompt,
                        reflections=reflections, search_round=rnd, pipe=pipe, topk=search_branch,
                        root_dir=outpath, config=config,
                        sample_path_lastround=dirs["samples_lastround"],
                        sample_path_best=dirs["samples_best"],
                        sample_path_bestround=dirs["samples_path_bestround"],
                        imagetoupdate=imagetoupdate, midimg_path=dirs["midimg"],
                        tag=meta0.get("tag"), total_rounds=search_rounds, chains=chains,
                        verifier=verifier, reflector=reflector, ctx=ctx, defer_saves=True, **hooks)
            if use_reflection:
                reflections = dp["reflections"]
            if use_refine:
                updated_prompt = dp["refined_prompt"]
            imagetoupdate = dp["generated"]
            chains = dp["chains"]
            if dp["flag_terminated"]:
                break
    flush_saves()
    ctx.barrier()
    return 0


def load_round0(paths: List[str], ctx: DistCtx) -> List[Candidate]:
    """Round-0 candidates of the noise-scaling stage, in name order like the reference's listing
    (tts_reflectionflow.py:537-547): `<k>_round@<seed>.latent.pt` as written by this framework (packed final latent,
    decoded on demand), or — a stage-0 directory produced by the REFERENCE — plain `<k>_round@<seed>.png` files,
    loaded as pixels (round-0 images are only scored and turned into condition images, never denoised further, so no
    latent is needed; verifiers that score latents cannot be used on them)."""
    stems = {}
    for p in paths:
        if p.endswith(".latent.pt"):
            stems.setdefault(p[: -len(".latent.pt")], {})["lat"] = p
        elif p.endswith(".png"):
            stems.setdefault(p[:-4], {})["png"] = p
    cands = []
    for stem in sorted(stems, key=lambda s: s + ".png"):
        name = os.path.basename(stem)
        seed = int(name.split("@")[-1]) if "@" in name and name.split("@")[-1].isdigit() else 0
        if "lat" in stems[stem]:
            lat = torch.load(stems[stem]["lat"], map_location="cpu").to(ctx.device)
            cands.append(Candidate(stem + ".png", seed, latents=lat))
        else:
            import numpy as np
            from PIL import Image
            with Image.open(stems[stem]["png"]) as im:
                u8 = torch.from_numpy(np.array(im.convert("RGB"))).to(ctx.device)
            cands.append(Candidate(stem + ".png", seed, image_u8=u8))
    if not cands:
        raise RuntimeError("no round-0 candidates (*.latent.pt or *.png) found under --imgpath")
    return cands


if __name__ == "__main__":
    raise SystemExit(main())
