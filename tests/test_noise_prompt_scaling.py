"""not-gpu: host logic of the noise + prompt-refinement search (reflectionflow_b200/tts/noise_prompt_scaling.py,
mirror of tts/tts_t2i_noise_prompt_scaling.py).  The pipeline is a cheap pure function (test-only) so that the round
logic — sharding, exchanges, the reference's ranking rules, the refiner hook, the artefact layout — runs on CPU,
single-process and under gloo with world_size 2."""
import json
import os
import socket
import sys

import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from reflectionflow_b200.pipeline import FluxPipelineOutput  # noqa: E402
from reflectionflow_b200.tts import noise_prompt_scaling as NP  # noqa: E402
from reflectionflow_b200.tts import search as S  # noqa: E402
from reflectionflow_b200.tts.dist import DistCtx  # noqa: E402
from reflectionflow_b200.tts.utils import get_noises  # noqa: E402
from reflectionflow_b200.tts.verifiers import (OpenAIShapedReflector, OpenAIShapedVerifier, StubReflector,  # noqa: E402
                                               StubVerifier)

H = W = 64
CONFIG = {
    "pipeline_args": {"pretrained_model_name_or_path": "black-forest-labs/FLUX.1-dev", "torch_dtype": "bf16",
                      "height": H, "width": W, "guidance_scale": 3.5, "num_inference_steps": 4},
    "verifier_args": {"name": "nvila"},
    "refine_args": {"choice_of_metric": "overall_score"},
    "search_args": {"search_branch": 5, "search_rounds": 3},
    "batch_size_for_img_gen": 2,
}


class FakePipe:
    """test-only stand-in for B200FluxPipeline.__call__: deterministic function of (noise, prompt)"""
    vae = None
    calls = 0

    def __call__(self, prompt=None, latents=None, guidance_scale=None, num_inference_steps=None, height=None,
                 width=None, output_type="pil"):
        assert output_type == "latent" and len(prompt) == latents.shape[0]
        assert (guidance_scale, num_inference_steps, height, width) == (3.5, 4, H, W)
        FakePipe.calls += 1
        out = []
        for p, x in zip(prompt, latents):
            h = sum(ord(c) for c in p) % 97 / 97.0
            out.append(0.5 * x.float() + 0.01 * h)
        return FluxPipelineOutput(images=torch.stack(out).to(torch.bfloat16))


class CountingRefiner(StubReflector):
    """rewrites every prompt with its round and position, so that the next round's prompts differ per candidate"""

    def __init__(self):
        self.seen = []

    def refine_prompt(self, cands, original_prompt, current_prompts, reflections, evaluations=None):
        self.seen.append((len(cands), list(current_prompts), reflections, evaluations))
        return [f"{original_prompt} / v{len(self.seen)}.{i}" for i, _ in enumerate(cands)]


def run_rounds(ctx, tmp):
    torch.manual_seed(4321)
    rounds, branch = CONFIG["search_args"]["search_rounds"], CONFIG["search_args"]["search_branch"]
    mid = os.path.join(tmp, "samples")
    if ctx.rank == 0:
        os.makedirs(mid, exist_ok=True)
    ctx.barrier()
    prompts = ["a photo of a dog"] * branch
    refiner, log = CountingRefiner(), []
    for rnd in range(1, rounds + 1):
        noises = get_noises(S.MAX_SEED, branch, H, W)
        dp = NP.sample(noises, "a photo of a dog", prompts, rnd, FakePipe(), branch, tmp, CONFIG, mid, tag="single",
                       verifier=StubVerifier("nvila"), refiner=refiner, ctx=ctx)
        prompts = dp["refined_prompt"]
        log.append({"topk_idx": dp["topk_idx"], "seeds": [c.seed for c in dp["generated"]],
                    "scores": [(o["label"], o["score"]) for o in dp["scores"]], "prompts": prompts,
                    "lat_sum": [float(c.latents.float().sum()) for c in dp["generated"]]})
    return {"log": log, "refiner_calls": len(refiner.seen)}


def test_single_process_rounds_follow_the_reference(tmp_path):
    res = run_rounds(DistCtx(), str(tmp_path))
    assert len(res["log"]) == 3 and res["refiner_calls"] == 3
    for r, entry in enumerate(res["log"], start=1):
        assert sorted(entry["topk_idx"]) == list(range(5))            # topk == search_branch: a permutation
        # the reference's nvila key: "yes" first by descending score, then "no" by ascending score (:113-118)
        key = lambda t: (0, -t[1]) if t[0] == "yes" else (1, t[1])
        ranked = [entry["scores"][i] for i in entry["topk_idx"]]
        assert ranked == sorted(entry["scores"], key=key)
        assert entry["prompts"] == [f"a photo of a dog / v{r}.{i}" for i in range(5)]
    # artefacts: NNNNN/samples/<round>_round@<seed>.*, refined_prompt<r> lines in best_img_meta.jsonl (:139-140)
    files = sorted(os.listdir(tmp_path / "samples"))
    assert len(files) == 15 and all("_round@" in f for f in files)
    lines = open(tmp_path / "best_img_meta.jsonl").read().strip().splitlines()
    assert [ln.split(":")[0] for ln in lines] == ["refined_prompt1", "refined_prompt2", "refined_prompt3"]
    assert json.loads(lines[1].split(": ", 1)[1]) == res["log"][1]["prompts"]


def test_datapoint_has_the_reference_keys_and_batches(tmp_path):
    torch.manual_seed(1)
    FakePipe.calls = 0
    os.makedirs(tmp_path / "samples")
    noises = get_noises(S.MAX_SEED, 5, H, W)
    dp = NP.sample(noises, "p", "p", 1, FakePipe(), 3, str(tmp_path), CONFIG, str(tmp_path / "samples"))
    for k in ("original_prompt", "refined_prompt", "search_round", "num_noises", "choice_of_metric"):  # :142-148
        assert k in dp
    assert dp["num_noises"] == 5 and len(dp["refined_prompt"]) == 5 and len(dp["topk_idx"]) == 3
    assert FakePipe.calls == 3  # batch_size_for_img_gen = 2 -> batches of 2, 2, 1 (:62-79)
    with pytest.raises(ValueError):
        NP.sample(noises, "p", ["p"] * 4, 1, FakePipe(), 3, str(tmp_path), CONFIG, str(tmp_path / "samples"))


def _fake_pixels(pipe, cand, height, width):
    """test-only decoder: a uint8 image that is a fixed function of the latent"""
    if cand.image_u8 is None:
        v = cand.latents.float().reshape(-1)[: 3 * 8 * 8]
        cand.image_u8 = ((v - v.min()) / (v.max() - v.min() + 1e-6) * 255).to(torch.uint8).reshape(8, 8, 3)
    return cand.image_u8


def test_openai_shaped_hooks_get_the_reference_messages(tmp_path):
    """verifier 'openai': ranking by [metric]['score'] descending, the refiner receives image + evaluation + original
    + current prompt (openai_verifier.py:300-317 as called from tts_t2i_noise_prompt_scaling.py:128-131)"""
    from tests.test_verifier_adapters import FakeOpenAI
    torch.manual_seed(2)
    os.makedirs(tmp_path / "samples")
    cfg = dict(CONFIG, verifier_args={"name": "openai"}, batch_size_for_img_gen=1)
    client = FakeOpenAI()
    ver = OpenAIShapedVerifier(client, "grade the image")
    ref = OpenAIShapedReflector(client, "write a reflection", "refine the prompt")
    noises = get_noises(S.MAX_SEED, 3, H, W)
    dp = NP.sample(noises, "a red cube", ["a red cube"] * 3, 1, FakePipe(), 3, str(tmp_path), cfg,
                   str(tmp_path / "samples"), tag=None, verifier=ver, refiner=ref, pixels_fn=_fake_pixels)
    scores = [o["overall_score"]["score"] for o in dp["scores"]]
    assert [scores[i] for i in dp["topk_idx"]] == sorted(scores, reverse=True)
    assert len(dp["refined_prompt"]) == 3 and all(isinstance(p, str) and p for p in dp["refined_prompt"])
    assert len(client.parse_calls) == 3  # one grading call per image, against the ORIGINAL prompt
    assert all(m[1]["content"][0] == {"type": "text", "text": "a red cube"} for _, m, _ in client.parse_calls)
    refine_calls = [m for _, m in client.create_calls if m[0]["content"] == "refine the prompt"]
    assert len(refine_calls) == 3
    kinds = [part["type"] for part in refine_calls[0][1]["content"]]
    texts = [part.get("text", "") for part in refine_calls[0][1]["content"]]
    assert kinds.count("image_url") == 1
    assert any(t.startswith("Original prompt: a red cube") for t in texts)
    assert any(t.startswith("Current prompt: a red cube") for t in texts)
    assert any(t.startswith("Evaluation of the generated images: {") for t in texts)
    assert os.path.exists(tmp_path / "samples" / os.path.basename(dp["generated"][0].name))  # PNG written


def _worker(rank, world, port, base, q):
    os.makedirs(base, exist_ok=True)
    os.chdir(base)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    res = run_rounds(DistCtx(rank, world, "cpu"), "run")
    q.put((rank, json.dumps(res)))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_world2_gloo_matches_single_process(tmp_path):
    os.makedirs(tmp_path / "w1", exist_ok=True)
    cwd = os.getcwd()
    os.chdir(tmp_path / "w1")
    try:
        single = run_rounds(DistCtx(), "run")
    finally:
        os.chdir(cwd)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, str(tmp_path / "w2"), q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=240) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    r0, r1 = json.loads(got[0]), json.loads(got[1])
    # every rank holds the same records / prompts; only rank 0 talks to the refiner
    assert r0["log"] == r1["log"] and (r0["refiner_calls"], r1["refiner_calls"]) == (3, 0)
    assert r0["log"] == json.loads(json.dumps(single))["log"], "sharded run differs from the single-process run"


def test_main_writes_the_reference_layout(tmp_path, monkeypatch):
    """main(): NNNNN/{metadata.jsonl, samples/<round>_round@<seed>.*, best_img_meta.jsonl} per metadata line
    (tts_t2i_noise_prompt_scaling.py:206-245), start/end index slicing, the refined prompts of round r feeding
    round r + 1.  The pipeline builder is replaced by the test-only FakePipe (no GPU here)."""
    cfg = dict(CONFIG, search_args={"search_branch": 3, "search_rounds": 2})
    (tmp_path / "cfg.json").write_text(json.dumps(cfg))
    metas = [{"prompt": f"a photo of object {i}", "tag": "single_object"} for i in range(3)]
    (tmp_path / "meta.jsonl").write_text("\n".join(json.dumps(m) for m in metas) + "\n")
    built = []

    def fake_build(config, args, ctx):
        built.append(config["pipeline_args"].get("lora_path", "absent"))
        return FakePipe()
    monkeypatch.setattr(NP, "build_pipeline", fake_build)
    out = tmp_path / "out"
    rc = NP.main(["--pipeline_config_path", str(tmp_path / "cfg.json"), "--meta_path", str(tmp_path / "meta.jsonl"),
                  "--output_dir", str(out), "--synthetic", "--seed", "11", "--start_index", "1"], ctx=DistCtx())
    assert rc == 0 and built == [None]  # entry A: the pipeline is built without the reflection LoRA
    assert sorted(os.listdir(out)) == ["00001", "00002"]
    for d, m in zip(("00001", "00002"), metas[1:]):
        assert json.load(open(out / d / "metadata.jsonl")) == m
        files = os.listdir(out / d / "samples")
        assert len(files) == 6 and sorted({f.split("_round@")[0] for f in files}) == ["1", "2"]
        lines = open(out / d / "best_img_meta.jsonl").read().strip().splitlines()
        assert [ln.split(":")[0] for ln in lines] == ["refined_prompt1", "refined_prompt2"]
        assert all(m["prompt"] in p for p in json.loads(lines[0].split(": ", 1)[1]))


@pytest.mark.parametrize("cfg_name", ["flux.1_dev_nvilascore.json", "flux.1_dev_gptscore.json"])
def test_main_runs_on_the_reference_config_files_unchanged(tmp_path, monkeypatch, cfg_name):
    """the reference's own tts/configs/*.json (1024x1024, 16 rounds x 2 candidates; copies stored under
    tests/golden/) drive main() as they are"""
    ref_cfg = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_configs", cfg_name)

    class AnySizePipe:
        vae = None

        def __call__(self, prompt=None, latents=None, output_type="pil", **kw):
            assert output_type == "latent" and latents.shape[1:] == (4096, 64) and kw["height"] == kw["width"] == 1024
            return FluxPipelineOutput(images=(latents.float() * 0.5).to(torch.bfloat16))

    monkeypatch.setattr(NP, "build_pipeline", lambda config, args, ctx: AnySizePipe())
    (tmp_path / "meta.jsonl").write_text(json.dumps({"prompt": "a photo of a clock", "tag": "single_object"}) + "\n")
    out = tmp_path / "out"
    assert NP.main(["--pipeline_config_path", ref_cfg, "--meta_path", str(tmp_path / "meta.jsonl"), "--output_dir",
                    str(out), "--synthetic", "--seed", "3"], ctx=DistCtx()) == 0
    cfg = json.load(open(ref_cfg))
    rounds, branch = cfg["search_args"]["search_rounds"], cfg["search_args"]["search_branch"]
    files = os.listdir(out / "00000" / "samples")
    assert len(files) == rounds * branch and {int(f.split("_round@")[0]) for f in files} == set(range(1, rounds + 1))
    lines = open(out / "00000" / "best_img_meta.jsonl").read().strip().splitlines()
    assert len(lines) == rounds and lines[-1].startswith(f"refined_prompt{rounds}: ")
