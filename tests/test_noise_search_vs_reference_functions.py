"""not-gpu: the two noise-search rounds against the reference's own unmodified functions, compiled out of their files
with `ast` and run over fakes (same method as tests/test_outer_loop_vs_reference_function.py):

* `tts/tts_t2i_noise_scaling.py::sample` (:16-77)   vs  reflectionflow_b200/tts/noise_scaling.py::sample
* `tts/tts_t2i_noise_prompt_scaling.py::sample` (:22-145)  vs  reflectionflow_b200/tts/noise_prompt_scaling.py::sample

Compared: what the pipeline is called with (prompts per batch, the stacked latents bit for bit, guidance / steps /
size), the file every image is written to, the returned datapoint, and for the prompt-refinement search the ranking,
the refined prompts and `best_img_meta.jsonl`.  What the reference's functions produced is stored under tests/golden/reference/ (tests/_refgold.py)."""
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
from reflectionflow_b200.tts import noise_prompt_scaling as NP  # noqa: E402
from reflectionflow_b200.tts import noise_scaling as NS  # noqa: E402
from reflectionflow_b200.tts.dist import DistCtx  # noqa: E402
from reflectionflow_b200.tts.utils import get_noises  # noqa: E402

from tests._refgold import Store, norm, ref_path  # noqa: E402

REF_NS = ref_path("tts/tts_t2i_noise_scaling.py")
REF_NP = ref_path("tts/tts_t2i_noise_prompt_scaling.py")
GOLD = Store("noise_search")

H = W = 64
CONFIG = {"pipeline_args": {"height": H, "width": W, "guidance_scale": 3.5, "num_inference_steps": 4},
          "verifier_args": {"name": "nvila"},
          "refine_args": {"choice_of_metric": "overall_score", "max_new_tokens": 64, "refine_prompt_relpath": "r.txt",
                          "reflexion_prompt_relpath": "x.txt", "verifier_prompt_relpath": "v.json"},
          "batch_size_for_img_gen": 2}


def _h(*parts) -> str:
    return hashlib.sha256("|".join(str(p) for p in parts).encode()).hexdigest()[:8]


def _compile(path, name, ns):
    fn = next(n for n in ast.parse(open(path).read()).body if isinstance(n, ast.FunctionDef) and n.name == name)
    exec(compile(ast.Module([fn], []), path, "exec"), ns)
    return ns[name]


class _Img:
    def __init__(self, log):
        self.log, self.src = log, None

    def save(self, path):
        self.src = self.src or path
        self.log.append(path)


class _RefPipe:
    """the reference calls pipe(prompt=, latents=, guidance_scale=, num_inference_steps=, height=, width=)"""

    def __init__(self):
        self.calls, self.saves = [], []

    def __call__(self, prompt, latents, guidance_scale, num_inference_steps, height, width):
        self.calls.append({"prompts": list(prompt), "latents": latents.clone(), "guidance_scale": guidance_scale,
                           "num_inference_steps": num_inference_steps, "height": height, "width": width})
        return FluxPipelineOutput(images=[_Img(self.saves) for _ in prompt])


class _OurPipe:
    vae = None

    def __init__(self):
        self.calls = []

    def __call__(self, prompt, latents, guidance_scale, num_inference_steps, height, width, output_type):
        assert output_type == "latent"
        self.calls.append({"prompts": list(prompt), "latents": latents.clone(), "guidance_scale": guidance_scale,
                           "num_inference_steps": num_inference_steps, "height": height, "width": width})
        return FluxPipelineOutput(images=(latents.float() * 0.5).to(torch.bfloat16))


def _calls(calls):
    """pipeline calls as stored: the latents by shape, dtype and a digest of their bytes"""
    out = []
    for c in calls:
        lat = c["latents"].contiguous()
        digest = hashlib.sha256(lat.view(torch.uint8).numpy().tobytes() if lat.dtype != torch.bfloat16
                                else lat.view(torch.int16).numpy().tobytes()).hexdigest()
        out.append(norm(dict({k: v for k, v in c.items() if k != "latents"},
                             latents=[list(lat.shape), str(lat.dtype), digest])))
    return out


def _same_calls(stored, ours):
    assert stored == _calls(ours)


def test_noise_scaling_round_equals_the_reference_function(tmp_path):
    torch.manual_seed(8)
    noises = get_noises(2 ** 31 - 1, 5, H, W)
    prompts = [f"a photo of a bench, variant {i}" for i in range(5)]
    mid = str(tmp_path / "samples")
    os.makedirs(mid)

    def reference_round():
        ref_sample = _compile(REF_NS, "sample", dict(torch=torch, DiffusionPipeline=object, copy=copy, os=os))
        rp = _RefPipe()
        dp = ref_sample(noises, prompts, 3, rp, CONFIG, "a photo of a bench", str(tmp_path / "ref_samples"))
        return {"calls": _calls(rp.calls), "saves": [os.path.basename(p) for p in rp.saves], "dp": dp}

    ref = GOLD.value("noise_scaling", reference_round)
    op = _OurPipe()
    our_dp = NS.sample(noises, prompts, 3, op, CONFIG, "a photo of a bench", mid, ctx=DistCtx())
    NS.flush_saves()
    _same_calls(ref["calls"], op.calls)                              # batches of 2, 2, 1; stacked latents identical
    assert [c["latents"].shape[0] for c in op.calls] == [2, 2, 1]
    assert [os.path.basename(p) for p in our_dp["generated_img"]] == ref["saves"]  # <round>_round@<seed>.png
    assert all(os.path.dirname(p) == mid for p in our_dp["generated_img"])
    assert norm({k: our_dp[k] for k in ref["dp"]}) == ref["dp"]       # prompt, search_round, num_noises
    assert sorted(os.listdir(mid)) == sorted(p[:-4] + ".latent.pt" for p in ref["saves"])


def _verdict(path):
    v = int(_h("score", os.path.basename(path)), 16)
    return ("yes" if v % 3 else "no"), float(np.float32(0.5 + (v % 1000) / 2000.0))


def _refined(original, path, evaluation, current):
    return f"{original} ~" + _h(os.path.basename(path), evaluation, current)


@pytest.mark.parametrize("seed", [0, 1])
def test_noise_prompt_scaling_rounds_equal_the_reference_function(tmp_path, seed):
    class ImageMod:
        @staticmethod
        def open(path):
            return path

    class Verifier:
        @staticmethod
        def generate_content(parts):
            label, score = _verdict(parts[0])
            logits = torch.zeros(1, 2)
            logits[0, 0 if label == "yes" else 1] = score
            return label, (logits,)

    class OpenAIVerifier:
        def __init__(self, **kw):
            pass

        def prepare_refine_prompt_inputs(self, images, original_prompt, current_prompt, evaluations=None):
            ev = evaluations if evaluations is not None else [None] * len(images)
            return list(zip(original_prompt, [im.src for im in images], ev, current_prompt))

        def refine_prompt(self, inputs):
            return [_refined(*item) for item in inputs]


    class OurVerifier:
        needs_images = False

        def score(self, cands, prompts, tag=None):
            return [dict(zip(("image_name", "label", "score"), (c.name,) + _verdict(c.name))) for c in cands]

    class OurRefiner:
        needs_images = False

        def refine_prompt(self, cands, original_prompt, current_prompts, reflections, evaluations=None):
            ev = evaluations if evaluations is not None else [None] * len(cands)
            return [_refined(original_prompt, c.name, e, cp) for c, e, cp in zip(cands, ev, current_prompts)]

    rounds, branch = 3, 5
    torch.manual_seed(40 + seed)
    noises = [get_noises(2 ** 31 - 1, branch, H, W) for _ in range(rounds)]
    logs = {}
    cwd = os.getcwd()

    def run(side):
        os.makedirs(tmp_path / side / "run" / "samples")
        os.chdir(tmp_path / side)
        try:
            prompts, log = ["a green bench"] * branch, []
            pipe = _RefPipe() if side == "ref" else _OurPipe()
            if side == "ref":
                ref_sample = _compile(REF_NP, "sample", dict(
                    torch=torch, Union=Union, List=List, Optional=Optional, DiffusionPipeline=object, copy=copy,
                    json=json, os=os, time=time, Image=ImageMod, OpenAIVerifier=OpenAIVerifier, verifier=Verifier,
                    yes_id=0, no_id=1))
            for rnd in range(1, rounds + 1):
                n0 = len(pipe.calls)
                if side == "ref":
                    dp = ref_sample(noises[rnd - 1], "a green bench", prompts, rnd, pipe, branch, "run", CONFIG,
                                    "run/samples", tag="colors")
                else:
                    dp = NP.sample(noises[rnd - 1], "a green bench", prompts, rnd, pipe, branch, "run", CONFIG,
                                   "run/samples", tag="colors", verifier=OurVerifier(), refiner=OurRefiner(),
                                   ctx=DistCtx())
                prompts = dp["refined_prompt"]
                log.append({"dp": norm({k: dp[k] for k in ("original_prompt", "refined_prompt", "search_round",
                                                           "num_noises", "choice_of_metric")}),
                            "calls": _calls(pipe.calls[n0:])})
        finally:
            os.chdir(cwd)
        return {"log": log, "meta": open(tmp_path / side / "run" / "best_img_meta.jsonl").read()}

    ref = GOLD.value(f"noise_prompt_scaling/seed{seed}", lambda: run("ref"))
    ours = run("ours")
    assert len(ref["log"]) == len(ours["log"]) == rounds
    for a, b in zip(ref["log"], ours["log"]):
        assert a["dp"] == b["dp"]
        assert a["calls"] == b["calls"]
    assert ref["meta"] == ours["meta"]
