"""not-gpu: the whole reflection round, `reflectionflow_b200.tts.reflectionflow.sample`, against the reference's own
UNMODIFIED `sample()` (tts/tts_reflectionflow.py:94-463).

The reference function is compiled out of its source file with `ast` and run with every external dependency faked:
`Image` (open / resize / save only record paths), the NVILA verifier (label and score are a hash of the image
path), `OpenAIVerifier` (reflections and refined prompts are hashes of exactly the fields the reference hands it),
`Condition` and `generate` (record their arguments; generated images take their identity from the file they are first
saved under).  The re-hosted loop gets the same scores and texts through its hooks and a latent-producing fake
denoiser.  Compared over several rounds with the reference's nvila and gptscore configurations (the latter also with
EQUAL grading dicts for different images, where `outputs.index` collapses them, App. B.7): the selected parents, the
prompt + " [Reflexion]: " + reflection strings and conditions handed to `generate`, the refined prompts / reflections
carried to the next round, the chains, `best_img_detailedscore.jsonl` and `best_img_meta.jsonl` byte for byte, and
which candidate lands in samples_lastround / samples_path_bestround / samples_best.  What the reference's function produced is stored under tests/golden/reference/ (tests/_refgold.py)."""
import ast
import copy
import hashlib
import json
import os
import sys
import time
from typing import List, Optional, Union

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from reflectionflow_b200.pipeline import FluxPipelineOutput  # noqa: E402
from reflectionflow_b200.tts import reflectionflow as RF  # noqa: E402
from reflectionflow_b200.tts.dist import DistCtx  # noqa: E402
from reflectionflow_b200.tts.utils import get_noises  # noqa: E402
from reflectionflow_b200.tts.verifiers import Candidate  # noqa: E402

from tests._refgold import Store, norm, ref_path  # noqa: E402

REF = ref_path("tts/tts_reflectionflow.py")
GOLD = Store("outer_loop")

H = W = 64
COND = 32


def _h(*parts) -> str:
    return hashlib.sha256("|".join(str(p) for p in parts).encode()).hexdigest()[:8]


def _verdict(image_id: str):
    """the fake NVILA: label and score from the image path alone (score float32-exact, as the reference reads
    a float32 logit)"""
    v = int(_h("score", os.path.basename(image_id)), 16)
    label = "yes" if v % 3 else "no"
    return label, float(np.float32(0.5 + (v % 1000) / 2000.0))


def _grading(image_id: str, unique: bool):
    """the fake GPT grader (openai_verifier.py:122-147 returns the bare model dump): few distinct scores; with
    `unique=False` the explanations are constant too, so different images get EQUAL dicts — the case in which the
    reference's `outputs.index` picks the first of them for all (App. B.7)"""
    v = int(_h("grade", os.path.basename(image_id)), 16)
    why = f"because {v % 97}" if unique else "ok"
    return {"accuracy_to_prompt": {"score": v % 3 + 6, "explanation": why},
            "overall_score": {"score": v % 4 + 4, "explanation": why}}


def _reflection(image_id, evaluation, current_prompt, reflection):
    return "fix-" + _h(os.path.basename(image_id), evaluation.replace(image_id, os.path.basename(image_id)),
                       current_prompt, reflection)


def _refined(original, image_id, evaluation, current_prompt, reflection):
    return f"{original} #" + _h(os.path.basename(image_id), evaluation, current_prompt, reflection)


# ------------------------------------------------------------------------------------------ reference side
class _Img:
    def __init__(self, world, src=None, resized=None):
        self.world, self.src, self.resized = world, src, resized

    def resize(self, size):
        return _Img(self.world, self.src, size)

    def save(self, path):
        if self.src is None:
            self.src = path  # a generated image is known by the file it is first written to
        self.world["saves"].append((path, self.src))


def _reference_sample(world):
    class ImageMod:
        Image = _Img

        @staticmethod
        def open(path):
            return _Img(world, path)

    class Verifier:
        @staticmethod
        def generate_content(parts):
            label, score = _verdict(parts[0].src)
            logits = torch.zeros(1, 2)
            logits[0, 0 if label == "yes" else 1] = score
            return label, (logits,)

        @staticmethod
        def prepare_inputs(images, prompts):
            return [im.src for im in images]

        @staticmethod
        def score(inputs, tag=None, max_new_tokens=None):
            return [_grading(src, world["unique"]) for src in inputs]

    class OpenAIVerifier:  # the reference builds its refiner from this name inside sample()
        def __init__(self, **kw):
            pass

        def prepare_reflexion_prompt_inputs(self, images, original_prompt, current_prompt, reflections, evaluations):
            return list(zip(images, evaluations, current_prompt, reflections))

        def generate_reflections(self, inputs, max_new_tokens=None):
            return [_reflection(*item) for item in inputs]

        def prepare_refine_prompt_inputs(self, images, original_prompt, current_prompt, reflections, evaluations=None):
            ev = evaluations if evaluations is not None else [None] * len(images)
            return list(zip(original_prompt, images, ev, current_prompt, reflections))

        def refine_prompt(self, inputs):
            return [_refined(*item) for item in inputs]

    class Condition:
        def __init__(self, condition, condition_type, position_delta):
            self.condition, self.condition_type, self.position_delta = condition, condition_type, position_delta

    def generate(pipe, prompt, conditions, height, width, model_config, default_lora):
        world["generate"].append({"prompts": list(prompt), "height": height, "width": width,
                                  "model_config": model_config, "default_lora": default_lora,
                                  "conditions": [(c.condition.src, c.condition.resized, c.condition_type,
                                                  [int(x) for x in c.position_delta]) for c in conditions]})
        return FluxPipelineOutput(images=[_Img(world) for _ in prompt])

    ns = dict(torch=torch, Union=Union, List=List, Optional=Optional, DiffusionPipeline=object, copy=copy, json=json,
              os=os, time=time, np=np, Image=ImageMod, OpenAIVerifier=OpenAIVerifier, Condition=Condition,
              generate=generate, verifier=Verifier, yes_id=0, no_id=1, MAX_RETRIES=5, RETRY_DELAY=0, client=None)
    fn = next(n for n in ast.parse(open(REF).read()).body if isinstance(n, ast.FunctionDef) and n.name == "sample")
    exec(compile(ast.Module([fn], []), REF, "exec"), ns)
    return ns["sample"]


# ------------------------------------------------------------------------------------------ re-hosted side
class _Verifier:
    needs_images = False

    def __init__(self, kind, unique):
        self.kind, self.unique = kind, unique

    def score(self, cands, prompts, tag=None):
        if self.kind == "openai":
            return [_grading(c.name, self.unique) for c in cands]
        out = []
        for c in cands:
            label, score = _verdict(c.name)
            out.append({"image_name": c.name, "label": label, "score": score})
        return out


class _Reflector:
    def generate_reflections(self, cands, original_prompt, current_prompts, reflections, evaluations):
        return [_reflection(c.name, ev, cp, rf) for c, ev, cp, rf in zip(cands, evaluations, current_prompts,
                                                                         reflections)]

    def refine_prompt(self, cands, original_prompt, current_prompts, reflections, evaluations=None):
        ev = evaluations if evaluations is not None else [None] * len(cands)
        return [_refined(original_prompt, c.name, e, cp, rf) for c, e, cp, rf in zip(cands, ev, current_prompts,
                                                                                      reflections)]


class _Pipe:
    vae = None


def _run_reference(tmp, config, rounds, branch, noises_per_round, unique):
    world = {"saves": [], "generate": [], "unique": unique}
    sample = _reference_sample(world)
    dirs = {k: os.path.join(tmp, k) for k in ("last", "best", "bestround", "mid")}
    for d in dirs.values():
        os.makedirs(d)
    parents = [f"r0/{i}.png" for i in range(branch)]
    upd, refl, chains, log = ["a photo of a cat"] * branch, [""] * branch, {}, []
    for rnd in range(1, rounds + 1):
        n_gen, n_sav = len(world["generate"]), len(world["saves"])
        dp = sample(noises_per_round[rnd - 1], "a photo of a cat", upd, refl, rnd, _Pipe(), branch, tmp, config,
                    dirs["last"], dirs["best"], dirs["bestround"], parents, dirs["mid"], rounds, chains, tag=None)
        parents, chains = dp["generated_img"], dp["chains"]
        upd, refl = dp["refined_prompt"], dp["reflections"]
        log.append({"dp": {k: dp[k] for k in ("generated_img", "refined_prompt", "reflections", "flag_terminated",
                                              "search_round", "num_noises", "choice_of_metric")},
                    "chains": copy.deepcopy(chains), "generate": world["generate"][n_gen:],
                    "saves": world["saves"][n_sav:]})
    return log


def _run_ours(tmp, config, rounds, branch, noises_per_round, unique):
    dirs = {k: os.path.join(tmp, k) for k in ("last", "best", "bestround", "mid")}
    for d in dirs.values():
        os.makedirs(d)
    g = torch.Generator().manual_seed(3)
    parents = [Candidate(f"r0/{i}.png", i, latents=torch.randn(1, 16, 64, generator=g).to(torch.bfloat16))
               for i in range(branch)]
    calls, by_latent = [], {}

    def condition_fn(pipe, parent, height, width, cond_size, seed):
        return {"src": parent.name, "resized": (cond_size, cond_size), "position_delta": [0, -cond_size // 16]}

    def generate_fn(pipe, prompt=None, conditions=None, latents=None, height=None, width=None, model_config=None,
                    default_lora=None, output_type=None):
        assert output_type == "latent" and len(prompt) == len(conditions) == 1
        calls.append({"prompts": list(prompt), "height": height, "width": width, "model_config": model_config,
                      "default_lora": default_lora,
                      "conditions": [(c["src"], c["resized"], "cot", c["position_delta"]) for c in conditions]})
        out = (latents.float() * 0.5 + len(calls)).to(torch.bfloat16)  # unique per call: identifies saved files
        return FluxPipelineOutput(images=out)

    upd, refl, chains, log = ["a photo of a cat"] * branch, [""] * branch, {}, []
    for rnd in range(1, rounds + 1):
        n_gen = len(calls)
        dp = RF.sample(noises_per_round[rnd - 1], "a photo of a cat", upd, refl, rnd, _Pipe(), branch, tmp, config,
                       dirs["last"], dirs["best"], dirs["bestround"], parents, dirs["mid"], rounds, chains, tag=None,
                       verifier=_Verifier(config["verifier_args"]["name"], unique), reflector=_Reflector(), ctx=DistCtx(), generate_fn=generate_fn,
                       condition_fn=condition_fn)
        for c in list(parents) + dp["generated"]:
            by_latent[c.latents.float().sum().item()] = c.name
        parents, chains = dp["generated"], dp["chains"]
        upd, refl = dp["refined_prompt"], dp["reflections"]
        files = {}
        for key in ("last", "best", "bestround"):
            for fn in sorted(os.listdir(dirs[key])):
                if fn.endswith(".latent.pt"):
                    lat = torch.load(os.path.join(dirs[key], fn))
                    files[f"{key}/{fn[:-len('.latent.pt')]}"] = by_latent[lat.float().sum().item()]
        log.append({"dp": {k: dp[k] for k in ("generated_img", "refined_prompt", "reflections", "flag_terminated",
                                              "search_round", "num_noises", "choice_of_metric")},
                    "chains": copy.deepcopy(chains), "generate": calls[n_gen:], "files": files})
    return log


@pytest.mark.parametrize("kind,unique", [("nvila", True), ("openai", True), ("openai", False)])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_reflection_rounds_equal_the_reference_function(tmp_path, seed, kind, unique):
    rounds, branch = 4, 4
    config = {"pipeline_args": {"height": H, "width": W, "condition_size": COND, "guidance_scale": 3.5,
                                "num_inference_steps": 4},
              "verifier_args": {"name": kind},
              "refine_args": {"choice_of_metric": "overall_score", "max_new_tokens": 1280,
                              "refine_prompt_relpath": "r.txt", "reflexion_prompt_relpath": "x.txt",
                              "verifier_prompt_relpath": "v.json"},
              "search_args": {"search_branch": branch, "search_rounds": rounds},
              "model": {"add_cond_attn": False, "latent_lora": False, "union_cond_attn": True},
              "reflection_args": {"run_reflection": True, "name": "openai"},
              "prompt_refiner_args": {"run_refinement": True}, "batch_size_for_img_gen": 1}
    torch.manual_seed(100 + seed)
    noises = [get_noises(2 ** 31 - 1, branch, H, W) for _ in range(rounds)]
    cwd = os.getcwd()

    def reference_run():  # the reference's unmodified sample() over the fakes, in its own directory
        os.makedirs(tmp_path / "ref")
        os.chdir(tmp_path / "ref")
        try:
            log = _run_reference("run", config, rounds, branch, noises, unique)
        finally:
            os.chdir(cwd)
        return {"log": log, "jsonl": {name: open(tmp_path / "ref" / "run" / name).read()
                                      for name in ("best_img_detailedscore.jsonl", "best_img_meta.jsonl")}}

    stored = GOLD.value(f"{kind}/unique{int(unique)}/seed{seed}", reference_run)
    try:  # our run writes relative artefact paths under its own directory
        os.makedirs(tmp_path / "ours")
        os.chdir(tmp_path / "ours")
        ours = _run_ours("run", config, rounds, branch, noises, unique)
    finally:
        os.chdir(cwd)
    ref = stored["log"]
    assert len(ref) == len(ours) == rounds
    for rnd, (a, b) in enumerate(zip(ref, ours), start=1):
        assert a["dp"] == norm(b["dp"]), f"round {rnd}: datapoint"
        assert a["chains"] == norm(b["chains"]), f"round {rnd}: chains"
        # the reference generates in batches of batch_size_for_img_gen = 1, in candidate order: same calls
        assert a["generate"] == norm(b["generate"]), f"round {rnd}: what the denoiser was asked for"
        # which candidate was written where (the reference names samples_best with a leaked loop index, App. B.9)
        ref_files = {}
        for dest, src in a["saves"]:
            key = os.path.basename(os.path.dirname(dest))
            if key in ("last", "bestround"):
                ref_files[f"{key}/{os.path.basename(dest)[:-4]}"] = src
            elif key == "best":
                ref_files["best/00000"] = src
        got = {k: v for k, v in b["files"].items()}
        if rnd > 1:  # files of earlier rounds stay on disk; the reference log holds this round's writes only
            got = {k: v for k, v in got.items() if k in ref_files}
        assert got == ref_files, f"round {rnd}: artefacts"
    for name, text in stored["jsonl"].items():
        assert text == open(tmp_path / "ours" / "run" / name).read(), name
