"""not-gpu: host logic of the sharded outer loop.  The denoiser is replaced by a cheap pure function
(`fake_generate`, test-only) so that the round logic — sharding, the per-round all-gather of score
records and parent latents, selection, chain bookkeeping, artefact layout — can run on CPU under
gloo with world_size 2 and be compared with the single-process result."""
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
from reflectionflow_b200.tts import reflectionflow as RF  # noqa: E402
from reflectionflow_b200.tts import search as S  # noqa: E402
from reflectionflow_b200.tts.dist import DistCtx  # noqa: E402
from reflectionflow_b200.tts.utils import get_noises  # noqa: E402
from reflectionflow_b200.tts.verifiers import Candidate, StubReflector, StubVerifier  # noqa: E402

H = W = 64  # 16 image tokens
CONFIG = {
    "pipeline_args": {"pretrained_model_name_or_path": "black-forest-labs/FLUX.1-dev",
                      "torch_dtype": "bf16", "height": H, "width": W, "condition_size": 32,
                      "guidance_scale": 3.5, "num_inference_steps": 4, "lora_path": "x"},
    "verifier_args": {"name": "nvila"},
    "refine_args": {"choice_of_metric": "overall_score"},
    "search_args": {"search_branch": 5, "search_rounds": 3},
    "model": {"add_cond_attn": False, "latent_lora": False, "union_cond_attn": True},
    "reflection_args": {"run_reflection": True, "name": "openai"},
    "prompt_refiner_args": {"run_refinement": True},
}


class FakePipe:
    vae = None


def fake_condition(pipe, parent, height, width, cond_size, seed):
    """test-only stand-in for decode -> resize -> encode (the product path needs the CUDA VAE):
    area-average of the parent's latent grid."""
    from reflectionflow_b200.pipeline import Condition
    lat = parent.latents
    b, n, c = lat.shape
    h, w = 2 * (height // 16), 2 * (width // 16)
    x = lat.float().view(b, h // 2, w // 2, c // 4, 2, 2).permute(0, 3, 1, 4, 2, 5).reshape(b, c // 4, h, w)
    ch = cond_size // 8
    x = torch.nn.functional.adaptive_avg_pool2d(x, (ch, ch))
    x = x.view(b, c // 4, ch // 2, 2, ch // 2, 2).permute(0, 2, 4, 1, 3, 5)
    return Condition("cot", latents=x.reshape(b, (ch // 2) ** 2, c).to(lat.dtype),
                     position_delta=[0, -cond_size // 16])


def fake_generate(pipe, prompt=None, conditions=None, latents=None, **kw):
    """test-only denoiser: deterministic function of (noise, parent condition, prompt)."""
    cond = conditions[0].latents.float()
    h = sum(ord(c) for c in prompt[0]) % 97 / 97.0
    out = 0.5 * latents.float() + 0.25 * cond.mean() + 0.01 * h
    out[..., : cond.shape[1] // 4, :] += 0.1 * cond[..., : cond.shape[1] // 4, :].mean()
    return FluxPipelineOutput(images=out.to(torch.bfloat16))


def run_rounds(ctx, tmp):
    torch.manual_seed(1234)
    rounds, branch = CONFIG["search_args"]["search_rounds"], CONFIG["search_args"]["search_branch"]
    g = torch.Generator().manual_seed(7)
    parents = [Candidate(f"r0/{i}.png", i, latents=torch.randn(1, 16, 64, generator=g).to(torch.bfloat16))
               for i in range(branch)]
    dirs = {k: os.path.join(tmp, k) for k in ("last", "best", "bestround", "mid")}
    if ctx.rank == 0:
        for d in dirs.values():
            os.makedirs(d, exist_ok=True)
    ctx.barrier()
    chains, log = {}, []
    upd, refl = ["a photo of a cat"] * branch, [""] * branch
    for rnd in range(1, rounds + 1):
        noises = get_noises(S.MAX_SEED, branch, H, W)
        dp = RF.sample(noises, "a photo of a cat", upd, refl, rnd, FakePipe(), branch, tmp, CONFIG,
                       dirs["last"], dirs["best"], dirs["bestround"], parents, dirs["mid"], rounds,
                       chains, verifier=StubVerifier("nvila"), reflector=StubReflector(), ctx=ctx,
                       generate_fn=fake_generate, condition_fn=fake_condition)
        parents, chains = dp["generated"], dp["chains"]
        upd, refl = dp["refined_prompt"], dp["reflections"]
        log.append({"topk_idx": dp["topk_idx"], "seeds": [c.seed for c in parents],
                    "scores": [(o["label"], o["score"]) for o in dp["scores"]],
                    "lat_sum": [float(c.latents.float().sum()) for c in parents]})
    return {"log": log, "chains": chains, "best": S.global_best(chains, "nvila")}


def _worker(rank, world, port, base, q):
    os.makedirs(base, exist_ok=True)
    os.chdir(base)  # artefact names (which seed the stub hooks) must not depend on the temp dir
    tmp = "run"
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    res = run_rounds(DistCtx(rank, world, "cpu"), tmp)
    q.put((rank, json.dumps(res)))
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_single_process_rounds(tmp_path):
    res = run_rounds(DistCtx(), str(tmp_path))
    assert len(res["log"]) == 3
    for r in res["log"]:
        assert sorted(set(r["topk_idx"])) == sorted(set(r["topk_idx"])) and len(r["topk_idx"]) == 5
    # artefacts follow the reference's layout
    mid = sorted(os.listdir(tmp_path / "mid"))
    assert len(mid) == 15 and all("_round@" in m for m in mid)
    assert os.path.exists(tmp_path / "best_img_meta.jsonl")
    lines = open(tmp_path / "best_img_detailedscore.jsonl").read().strip().splitlines()
    assert len(lines) == 3 and "filenames_batch" in json.loads(lines[0])
    assert len(os.listdir(tmp_path / "last")) == 5 and len(os.listdir(tmp_path / "best")) == 1
    # chains: 5 roots, every later candidate attached to exactly one chain (nvila break rule)
    assert len(res["chains"]) == 5
    assert sum(len(c["images"]) for c in res["chains"].values()) == 15


@pytest.mark.timeout(300)
def test_world2_gloo_matches_single_process(tmp_path):
    os.makedirs(tmp_path / "w1", exist_ok=True)
    cwd = os.getcwd()
    os.chdir(tmp_path / "w1")
    try:
        single = run_rounds(DistCtx(), "run")
    finally:
        os.chdir(cwd)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, str(tmp_path / "w2"), q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=240) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    r0, r1 = json.loads(got[0]), json.loads(got[1])
    assert r0 == r1, "ranks disagree"
    assert r0 == json.loads(json.dumps(single)), "sharded run differs from the single-process run"


def test_condition_needs_a_vae():
    """no latent-space stand-in in the product: without a VAE the parent condition raises"""
    lat = torch.randn(1, 16, 64).to(torch.bfloat16)
    with pytest.raises(RuntimeError, match="vae"):
        RF.parent_condition(FakePipe(), Candidate("x.png", 0, latents=lat), H, W, 32, 0)


class _FavourRound1(StubVerifier):
    """scores fall with the round number: the global best is a round-1 candidate"""

    def value(self, cand):
        rnd = int(os.path.basename(cand.name).split("_round@")[0]) if "_round@" in cand.name else 0
        return (0.05 / (1 + rnd) if rnd else -0.05) + 1e-4 * (cand.seed % 7)


def test_best_of_an_early_round_is_still_written(tmp_path):
    """ADVICE r01 (high): the global best of round 1 must reach samples_best/ after round 3."""
    torch.manual_seed(99)
    rounds, branch = 3, 4
    g = torch.Generator().manual_seed(3)
    parents = [Candidate(f"r0/{i}.png", i, latents=torch.randn(1, 16, 64, generator=g).to(torch.bfloat16))
               for i in range(branch)]
    tmp = str(tmp_path)
    dirs = {k: os.path.join(tmp, k) for k in ("last", "best", "bestround", "mid")}
    for d in dirs.values():
        os.makedirs(d)
    chains = {}
    upd, refl = ["p"] * branch, [""] * branch
    ver = _FavourRound1("nvila")
    for rnd in range(1, rounds + 1):
        noises = get_noises(S.MAX_SEED, branch, H, W)
        dp = RF.sample(noises, "p", upd, refl, rnd, FakePipe(), branch, tmp, CONFIG, dirs["last"],
                       dirs["best"], dirs["bestround"], parents, dirs["mid"], rounds, chains,
                       verifier=ver, reflector=StubReflector(), ctx=DistCtx(),
                       generate_fn=fake_generate, condition_fn=fake_condition)
        parents, chains = dp["generated"], dp["chains"]
        upd, refl = dp["refined_prompt"], dp["reflections"]
    best = S.global_best(chains, "nvila")
    assert os.path.basename(best).startswith("1_round@"), best
    files = os.listdir(dirs["best"])
    assert files == ["00000.latent.pt"], files
    want = torch.load(os.path.join(dirs["mid"], os.path.basename(best)[:-4] + ".latent.pt"))
    assert torch.equal(torch.load(os.path.join(dirs["best"], files[0])), want)
    assert len(os.listdir(dirs["bestround"])) == branch


class _OpenAIShaped(StubVerifier):
    def score_one(self, cand, prompt):
        v = self.value(cand)
        s = max(0, min(10, int(round(5 + 60.0 * v))))
        return {"accuracy_to_prompt": {"score": s, "explanation": f"why {cand.seed}"},
                "overall_score": {"score": s, "explanation": f"overall {cand.seed}"}}


def test_openai_shaped_outputs_travel_whole(tmp_path):
    """ADVICE r01 (medium): every aspect + explanation reaches the reflector and the jsonl."""
    torch.manual_seed(5)
    cfg = dict(CONFIG, verifier_args={"name": "openai"})
    g = torch.Generator().manual_seed(3)
    parents = [Candidate(f"r0/{i}.png", i, latents=torch.randn(1, 16, 64, generator=g).to(torch.bfloat16))
               for i in range(3)]
    tmp = str(tmp_path)
    dirs = {k: os.path.join(tmp, k) for k in ("last", "best", "bestround", "mid")}
    for d in dirs.values():
        os.makedirs(d)
    seen = {}

    class Refl(StubReflector):
        def generate_reflections(self, cands, op, cp, refl, evaluations):
            seen["ev"] = evaluations
            return super().generate_reflections(cands, op, cp, refl, evaluations)
    noises = get_noises(S.MAX_SEED, 3, H, W)
    RF.sample(noises, "p", ["p"] * 3, [""] * 3, 1, FakePipe(), 3, tmp, cfg, dirs["last"], dirs["best"],
              dirs["bestround"], parents, dirs["mid"], 2, {}, verifier=_OpenAIShaped("openai"),
              reflector=Refl(), ctx=DistCtx(), generate_fn=fake_generate, condition_fn=fake_condition)
    ev = [json.loads(e) for e in seen["ev"]]
    assert all("accuracy_to_prompt" in e and e["overall_score"]["explanation"].startswith("overall") for e in ev)
    line = json.loads(open(os.path.join(tmp, "best_img_detailedscore.jsonl")).readline())
    assert "accuracy_to_prompt" in line["evaluation"][0]


def test_image_consuming_hooks_get_pixels_of_latent_only_parents(tmp_path, monkeypatch):
    """An OpenAI-shaped reflection writer / refiner looks at the selected parents' images.  Parents loaded from
    `*.latent.pt` (round 0) or generated on another rank carry latents only: rank 0 decodes them before the hook,
    also when the verifier itself did not need pixels (stub / latent-space verifier)."""
    from tests.test_verifier_adapters import FakeOpenAI
    from reflectionflow_b200.tts.verifiers import OpenAIShapedReflector
    decoded = []

    def fake_pixels(pipe, cand, height, width):
        if cand.image_u8 is None:
            decoded.append(cand.name)
            v = cand.latents.float().reshape(-1)[:192]
            cand.image_u8 = ((v - v.min()) / (v.max() - v.min() + 1e-6) * 255).to(torch.uint8).reshape(8, 8, 3)
        return cand.image_u8
    monkeypatch.setattr(RF, "_ensure_pixels", fake_pixels)
    torch.manual_seed(5)
    branch = 3
    g = torch.Generator().manual_seed(1)
    parents = [Candidate(f"r0/{i}.png", i, latents=torch.randn(1, 16, 64, generator=g).to(torch.bfloat16))
               for i in range(branch)]
    tmp = str(tmp_path)
    dirs = {k: os.path.join(tmp, k) for k in ("last", "best", "bestround", "mid")}
    for d in dirs.values():
        os.makedirs(d)
    client = FakeOpenAI()
    refl = OpenAIShapedReflector(client, "REFLEX", "REFINE")
    cfg = dict(CONFIG, search_args={"search_branch": branch, "search_rounds": 2})
    dp = RF.sample(get_noises(S.MAX_SEED, branch, H, W), "a cat", ["a cat"] * branch, [""] * branch, 1, FakePipe(),
                   branch, tmp, cfg, dirs["last"], dirs["best"], dirs["bestround"], parents, dirs["mid"], 2, {},
                   verifier=StubVerifier("nvila"), reflector=refl, ctx=DistCtx(), generate_fn=fake_generate,
                   condition_fn=fake_condition)
    assert set(decoded) >= {p.name for p in parents}           # every selected parent was decoded for the hooks
    assert len(client.create_calls) == 2 * branch               # one reflection + one refinement request per parent
    assert all(m[1]["content"][-2]["type"] == "image_url" or any(p["type"] == "image_url" for p in m[1]["content"])
               for _, m in client.create_calls)
    assert len(dp["reflections"]) == branch and dp["reflections"][0].startswith("[REFLEX] Original prompt: a cat")
    assert dp["refined_prompt"][0].startswith("[REFINE] Original prompt: a cat")


def test_round0_from_a_reference_written_png_directory(tmp_path):
    """A stage-0 directory produced by the REFERENCE holds `samples/<k>_round@<seed>.png` only.  `load_round0` takes
    those as pixel-only candidates (name order, like the reference's listing); they can be scored and turned into
    conditions, and a directory written by this framework (PNG + packed latent) still loads the latents."""
    from PIL import Image
    samples = tmp_path / "samples"
    os.makedirs(samples)
    g = torch.Generator().manual_seed(4)
    seeds = [907, 15, 15002]
    for s in seeds:
        px = (torch.rand(16, 16, 3, generator=g) * 255).to(torch.uint8).numpy()
        Image.fromarray(px).save(samples / f"1_round@{s}.png")
    paths = sorted(str(samples / f) for f in os.listdir(samples))
    cands = RF.load_round0(paths, DistCtx())
    assert [c.seed for c in cands] == [15, 15002, 907] and all(c.latents is None and c.image_u8 is not None
                                                               for c in cands)
    assert [os.path.basename(c.name) for c in cands] == sorted(os.path.basename(p) for p in paths)
    outs = StubVerifier("nvila").score(cands, ["p"] * 3)
    assert len({o["score"] for o in outs}) == 3 and all(o["label"] in ("yes", "no") for o in outs)

    def pixel_condition(pipe, parent, height, width, cond_size, seed):
        from reflectionflow_b200.pipeline import Condition
        v = parent.image_u8.float().mean() / 255.0
        return Condition("cot", latents=torch.full((1, (cond_size // 16) ** 2, 64), float(v)).to(torch.bfloat16),
                         position_delta=[0, -cond_size // 16])

    dirs = {k: str(tmp_path / k) for k in ("last", "best", "bestround", "mid")}
    for d in dirs.values():
        os.makedirs(d)
    torch.manual_seed(0)
    dp = RF.sample(get_noises(S.MAX_SEED, 3, H, W), "a cat", ["a cat"] * 3, [""] * 3, 1, FakePipe(), 3, str(tmp_path),
                   dict(CONFIG, search_args={"search_branch": 3, "search_rounds": 2}), dirs["last"], dirs["best"],
                   dirs["bestround"], cands, dirs["mid"], 2, {}, verifier=StubVerifier("nvila"),
                   reflector=StubReflector(), ctx=DistCtx(), generate_fn=fake_generate, condition_fn=pixel_condition)
    assert len(dp["generated"]) == 3 and sorted(dp["topk_idx"]) == [0, 1, 2]
    # this framework's own stage-0 output: the latent next to the PNG wins
    torch.save(torch.randn(1, 16, 64).to(torch.bfloat16), samples / "1_round@15.latent.pt")
    again = RF.load_round0(sorted(str(samples / f) for f in os.listdir(samples)), DistCtx())
    assert [c.latents is not None for c in again] == [True, False, False] and len(again) == 3
    with pytest.raises(RuntimeError, match="no round-0"):
        RF.load_round0([str(tmp_path / "metadata.jsonl")], DistCtx())


def test_main_on_the_reference_config_and_a_reference_written_stage0(tmp_path, monkeypatch):
    """End to end on the host side: the reference's own `flux.1_dev_nvilascore.json` (1024x1024, condition 512, 16
    rounds x 2 candidates) and a stage-0 directory as the REFERENCE writes it (metadata.jsonl + samples/*.png) drive
    `reflectionflow.main`; denoiser and VAE are test-only fakes.  The artefact tree is the one `verifier_filter.py` and
    the GenEval tooling read (tts_reflectionflow.py:562-579, 398-448)."""
    from PIL import Image
    ref_cfg = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_configs", "flux.1_dev_nvilascore.json")
    stage0 = tmp_path / "stage0" / "00000"
    os.makedirs(stage0 / "samples")
    (stage0 / "metadata.jsonl").write_text(json.dumps({"prompt": "a photo of a kite", "tag": "single_object"}))
    g = torch.Generator().manual_seed(9)
    for s in (11, 22):
        Image.fromarray((torch.rand(32, 32, 3, generator=g) * 255).to(torch.uint8).numpy()).save(
            stage0 / "samples" / f"1_round@{s}.png")
    monkeypatch.setattr(RF, "build_pipeline", lambda config, args, ctx: FakePipe())

    def pixel_or_latent_condition(pipe, parent, height, width, cond_size, seed):
        from reflectionflow_b200.pipeline import Condition
        assert (height, width, cond_size) == (1024, 1024, 512)
        v = parent.image_u8.float().mean() / 255.0 if parent.latents is None else parent.latents.float().mean()
        return Condition("cot", latents=torch.full((1, 1024, 64), float(v)).to(torch.bfloat16),
                         position_delta=[0, -32])

    out = tmp_path / "stage1"
    rc = RF.main(["--pipeline_config_path", ref_cfg, "--imgpath", str(tmp_path / "stage0"), "--output_dir", str(out),
                  "--synthetic", "--seed", "5"], ctx=DistCtx(), generate_fn=fake_generate,
                 condition_fn=pixel_or_latent_condition)
    assert rc == 0
    cfg = json.load(open(ref_cfg))
    rounds, branch = cfg["search_args"]["search_rounds"], cfg["search_args"]["search_branch"]
    root = out / "00000"
    assert json.load(open(root / "metadata.jsonl"))["prompt"] == "a photo of a kite"
    mid = os.listdir(root / "midimg")
    assert len(mid) == rounds * branch and {int(f.split("_round@")[0]) for f in mid} == set(range(1, rounds + 1))
    assert len(os.listdir(root / "samples_lastround")) == branch
    assert len(os.listdir(root / "samples_path_bestround")) == branch and len(os.listdir(root / "samples_best")) == 1
    meta = open(root / "best_img_meta.jsonl").read().strip().splitlines()
    assert sum(ln.startswith("reflections") for ln in meta) == rounds
    assert sum(ln.startswith("refined_prompt") for ln in meta) == rounds
    assert sum(ln.startswith("filenames_batch") for ln in meta) == rounds
    assert len(open(root / "best_img_detailedscore.jsonl").read().strip().splitlines()) == rounds
