"""not-gpu: the verifier / reflector adapters (SURVEY §8 a11, f3) against fake external models with
the real call surfaces: NVILA `generate_content`, the OpenAI SDK's `beta.chat.completions.parse` /
`chat.completions.create`, and the Image-Verifier's `reward` — return schemas as the reference's
(tts_reflectionflow.py:157-170,345-352; verifiers/openai_verifier.py:23-164,241-317;
reward_modeling/inference.py:155-180), plus one outer-loop round driven by the "ours" branch."""
import json
import os
import types

import pytest
import torch
from PIL import Image

from reflectionflow_b200.tts import reflectionflow as RF
from reflectionflow_b200.tts import search as S
from reflectionflow_b200.tts import verifiers as V
from reflectionflow_b200.tts.dist import DistCtx
from reflectionflow_b200.tts.utils import get_noises


def _cand(i, colour):
    c = V.Candidate(f"mid/1_round@{i}.png", i, latents=torch.zeros(1, 16, 64, dtype=torch.bfloat16))
    c.image = Image.new("RGB", (32, 32), colour)
    return c


class FakeNvila:
    """generate_content([PIL, prompt]) -> (label, [logits[1, vocab]]) like the NVILA remote code"""

    def __init__(self):
        self.calls = []

    def generate_content(self, parts):
        im, prompt = parts
        self.calls.append((im.size, prompt))
        r = im.getpixel((0, 0))[0] / 255.0
        logits = torch.zeros(1, 10)
        logits[0, 3], logits[0, 7] = r, 1 - r  # yes_id = 3, no_id = 7
        return ("yes" if r >= 0.5 else "no"), [logits]


def test_nvila_adapter_schema_and_selection():
    cands = [_cand(0, (200, 0, 0)), _cand(1, (20, 0, 0)), _cand(2, (255, 0, 0))]
    m = FakeNvila()
    out = V.NvilaVerifier(m, yes_id=3, no_id=7).score(cands, ["a cat"] * 3)
    assert [o["label"] for o in out] == ["yes", "no", "yes"]
    assert all(set(o) == {"image_name", "label", "score"} and isinstance(o["score"], float) for o in out)
    assert out[0]["score"] == pytest.approx(200 / 255) and out[1]["score"] == pytest.approx(1 - 20 / 255)
    assert m.calls[0] == ((32, 32), "a cat")
    order = [o["image_name"] for o in S.sort_outputs(out, "nvila")]
    assert order == [cands[2].name, cands[0].name, cands[1].name]


def test_nvila_adapter_needs_pixels():
    c = V.Candidate("x.png", 0, latents=torch.zeros(1, 16, 64))
    with pytest.raises(RuntimeError, match="pixels"):
        V.NvilaVerifier(FakeNvila(), 3, 7).score([c], ["p"])


class FakeOpenAI:
    """the slice of the OpenAI SDK the reference uses"""

    def __init__(self):
        self.parse_calls, self.create_calls = [], []
        outer = self

        class _Parse:
            def parse(self, model, messages, temperature, response_format):
                outer.parse_calls.append((model, messages, response_format))
                n = len(messages[1]["content"][1]["image_url"]["url"])
                fields = {a: {"score": (n + k) % 11, "explanation": f"{a} because"}
                          for k, a in enumerate(response_format.model_fields)}
                parsed = response_format(**fields)
                return types.SimpleNamespace(choices=[types.SimpleNamespace(
                    message=types.SimpleNamespace(parsed=parsed))])

        class _Create:
            def create(self, model, messages, temperature):
                outer.create_calls.append((model, messages))
                txt = " | ".join(p["text"] for p in messages[1]["content"] if p["type"] == "text")
                return types.SimpleNamespace(choices=[types.SimpleNamespace(
                    message=types.SimpleNamespace(content=f"[{messages[0]['content']}] {txt}"))])
        self.beta = types.SimpleNamespace(chat=types.SimpleNamespace(completions=_Parse()))
        self.chat = types.SimpleNamespace(completions=_Create())


def test_openai_shaped_verifier_schema():
    cl = FakeOpenAI()
    instr = {"position": "grade position", "colors": "grade colours"}
    v = V.OpenAIShapedVerifier(cl, instr, model_name="m")
    cands = [_cand(0, (1, 2, 3)), _cand(1, (9, 9, 9))]
    out = v.score(cands, ["a red cube left of a ball"] * 2, tag="position")
    assert len(out) == len(cands)
    for o in out:
        assert set(o) == set(V.GRADING_ASPECTS["position"])   # the bare model dump, as upstream (:147)
        assert isinstance(o["overall_score"]["score"], int) and o["overall_score"]["explanation"]
    model, messages, fmt = cl.parse_calls[0]
    assert model == "m" and messages[0] == {"role": "system", "content": "grade position"}
    assert messages[1]["content"][0] == {"type": "text", "text": "a red cube left of a ball"}
    assert messages[1]["content"][1]["image_url"]["url"].startswith("data:image/jpeg;base64,")
    assert fmt.__name__ == "Grading_position"
    # general rubric: six aspects, plain-string system prompt
    v2 = V.OpenAIShapedVerifier(FakeOpenAI(), "general rubric")
    o2 = v2.score(cands[:1], ["p"])[0]
    assert set(o2) == set(V.GRADING_ASPECTS[None])
    assert S.metric_value(o2, "overall_score") == o2["overall_score"]["score"]


def test_openai_shaped_reflector_message_layout():
    cl = FakeOpenAI()
    r = V.OpenAIShapedReflector(cl, "REFLEX", "REFINE", model_name="m")
    cands = [_cand(0, (1, 2, 3)), _cand(1, (4, 5, 6))]
    refl = r.generate_reflections(cands, "orig", ["cur0", "cur1"], ["old0", "old1"], ["ev0", "ev1"])
    assert len(refl) == 2 and refl[0].startswith("[REFLEX] Original prompt: orig")
    assert "The updated prompt to generate the image is: cur1[Reflexion]: old1" in refl[1]
    assert "Evaluation of the generated image: ev1" in refl[1]
    ref = r.refine_prompt(cands, "orig", ["cur0", "cur1"], refl, None)
    assert ref[0].startswith("[REFINE] Original prompt: orig | Current prompt: cur0 | Reflection prompt: ")
    assert "Evaluation of the generated images" not in ref[0]
    ref2 = r.refine_prompt(cands, "orig", ["cur0", "cur1"], refl, ["e0", "e1"])
    assert "Evaluation of the generated images: e1" in ref2[1]
    assert ref2[1].endswith("Please refine the current prompt to improve the overall quality of the future "
                            "generated images.")


class FakeRewardModel:
    """reward_modeling/inference.py:155-180: reward(images, prompts, use_norm) -> [{'VQ','Overall'}]"""

    def __init__(self):
        self.batches = []

    def reward(self, images, prompts, max_pixels=None, use_norm=True):
        self.batches.append(len(images))
        out = []
        for im in images:
            vq = im.getpixel((0, 0))[1] / 64.0 - (1.0 if use_norm else 0.0)
            out.append({"VQ": vq, "Overall": vq})
        return out


def test_ours_branch_is_batched_and_metric_ordered():
    rm = FakeRewardModel()
    v = V.load_verifier({"name": "ours"}, synthetic=False, choice_of_metric="Overall", inferencer=rm)
    cands = [_cand(i, (0, 10 * i, 0)) for i in range(11)]
    out = v.score(cands, ["p"] * 11)
    assert rm.batches == [8, 3]
    assert out[3] == {"VQ": 30 / 64 - 1, "Overall": 30 / 64 - 1, "image_name": cands[3].name}
    best = S.sort_outputs(out, "ours", "Overall")[0]
    assert best["image_name"] == cands[10].name
    with pytest.raises(ValueError):
        V.load_verifier({"name": "gemini"}, synthetic=True)
    with pytest.raises(RuntimeError, match="inferencer"):
        V.load_verifier({"name": "ours"}, synthetic=False)


def test_outer_loop_round_with_the_ours_branch(tmp_path):
    """sample() end to end (CPU, fake denoiser) with verifier 'ours': scalar rewards travel through
    the record all-gather, the chains and the best-of bookkeeping."""
    from tests.test_outer_loop import CONFIG, FakePipe, fake_condition, fake_generate, H, W
    cfg = dict(CONFIG, verifier_args={"name": "ours"}, refine_args={"choice_of_metric": "Overall"})
    torch.manual_seed(11)
    g = torch.Generator().manual_seed(3)
    parents = [V.Candidate(f"r0/{i}.png", i, latents=torch.randn(1, 16, 64, generator=g).to(torch.bfloat16))
               for i in range(3)]
    tmp = str(tmp_path)
    dirs = {k: os.path.join(tmp, k) for k in ("last", "best", "bestround", "mid")}
    for d in dirs.values():
        os.makedirs(d)
    chains = {}
    upd, refl = ["p"] * 3, [""] * 3
    ver = V.StubVerifier("ours", "Overall")
    for rnd in (1, 2):
        dp = RF.sample(get_noises(S.MAX_SEED, 3, H, W), "p", upd, refl, rnd, FakePipe(), 3, tmp, cfg,
                       dirs["last"], dirs["best"], dirs["bestround"], parents, dirs["mid"], 2, chains,
                       verifier=ver, reflector=V.StubReflector(), ctx=DistCtx(),
                       generate_fn=fake_generate, condition_fn=fake_condition)
        parents, chains, upd, refl = dp["generated"], dp["chains"], dp["refined_prompt"], dp["reflections"]
        assert all(isinstance(o["Overall"], float) for o in dp["scores"])
    assert len(chains) == 3 and all(len(c["scores"]) >= 1 for c in chains.values())
    assert len(os.listdir(dirs["best"])) == 1
    line = json.loads(open(os.path.join(tmp, "best_img_detailedscore.jsonl")).readline())
    assert "Overall" in line["evaluation"][0]


def test_reflection_generator_ours_messages_and_retries(tmp_path):
    """tts_reflectionflow.py:26-44, 220-238: one request per image with the reference's two messages; failures are
    retried; refinement is delegated"""
    calls, fail = [], {"n": 2}

    class Client:
        class chat:  # noqa: N801 - mirrors the SDK attribute chain
            class completions:  # noqa: N801
                @staticmethod
                def create(messages, model):
                    calls.append((messages, model))
                    if fail["n"] > 0:
                        fail["n"] -= 1
                        raise ConnectionError("server busy")
                    return types.SimpleNamespace(choices=[types.SimpleNamespace(
                        message=types.SimpleNamespace(content=f"reflection #{len(calls)}"))])

    on_disk = _cand(0, (1, 2, 3))
    on_disk.name = str(tmp_path / "1_round@5.png")
    on_disk.pil().save(on_disk.name)
    in_memory = _cand(1, (4, 5, 6))
    r = V.ReflectionGeneratorOurs(Client(), retry_delay=0.0)
    out = r.generate_reflections([on_disk, in_memory], "a blue bird", ["cur"] * 2, [""] * 2, ["{}"] * 2)
    assert out == ["reflection #3", "reflection #4"] and len(calls) == 4      # two failures retried
    messages, model = calls[-2]
    assert model == "Qwen/Qwen2.5-VL-7B-Instruct" and messages[0] == {"role": "system",
                                                                     "content": "You are a helpful assistant."}
    assert messages[1]["content"][0] == {"type": "image_url", "image_url": {"url": on_disk.name}}
    assert messages[1]["content"][1]["text"] == ("Generate reflections to improve the input image according to the "
                                                 'prompt. The prompt is: "a blue bird"')
    assert calls[-1][0][1]["content"][0]["image_url"]["url"].startswith("data:image/jpeg;base64,")
    assert r.refine_prompt([on_disk], "p", ["cur"], out[:1]) == ["cur"]         # no refiner: prompts unchanged
    inner = V.StubReflector()
    assert V.ReflectionGeneratorOurs(Client(), refiner=inner).refine_prompt([on_disk], "p", ["cur"], out[:1]) == \
        inner.refine_prompt([on_disk], "p", ["cur"], out[:1])
    fail["n"] = 99
    with pytest.raises(ConnectionError):
        V.ReflectionGeneratorOurs(Client(), max_retries=2, retry_delay=0.0).generate_reflections(
            [in_memory], "p", ["c"], [""], ["{}"])


def test_grading_schemas_equal_the_reference_classes():
    """openai_verifier.py:23-69: every `Grading*` pydantic class of the reference, field for field and in order (read
    from the reference source when recording, tests/_refgold.py; the pinned table below as well)"""
    import ast
    pinned = {None: 6, "single_object": 4, "two_object": 4, "counting": 4, "colors": 4, "position": 4, "color_attr": 4}
    assert {k: len(v) for k, v in V.GRADING_ASPECTS.items()} == pinned
    for tag, aspects in V.GRADING_ASPECTS.items():
        model = V.grading_model(tag)
        assert tuple(model.model_fields) == tuple(aspects) and aspects[-1] == "overall_score"
        assert model.__name__ == ("Grading" if tag is None else f"Grading_{tag}")
        sub = model.model_fields["overall_score"].annotation
        assert tuple(sub.model_fields) == ("score", "explanation")
    from tests._refgold import Store, norm, ref_path

    def reference_classes():
        ref = {}
        for node in ast.parse(open(ref_path("tts/verifiers/openai_verifier.py")).read()).body:
            if isinstance(node, ast.ClassDef) and node.name.startswith("Grading"):
                tag = node.name[len("Grading_"):] or None
                ref[tag] = list(s.target.id for s in node.body if isinstance(s, ast.AnnAssign))
        return ref

    ref = Store("verifier_adapters").value("grading_schemas", reference_classes)
    assert ref == norm({k: list(v) for k, v in V.GRADING_ASPECTS.items()})


def test_message_builders_equal_the_reference_methods():
    """openai_verifier.py:90-118, 166-238, 256-293: the three `prepare_*` methods of the reference's OpenAIVerifier
    (they do not touch `self`), compiled out of the reference source and fed the same images / strings as the
    adapters here — the request payloads must be identical, JPEG bytes included (stored, tests/_refgold.py)."""
    import ast, base64
    from io import BytesIO
    from typing import Union
    from PIL import Image
    from tests._refgold import Store, norm, ref_path
    cands = [_cand(0, (200, 10, 30)), _cand(1, (5, 90, 250))]
    images = [c.pil() for c in cands]
    orig, cur = ["a red cube"] * 2, ["a red cube, studio light", "a red cube on a table"]
    refl, evals = ["make it redder", "center the cube"], ['{"overall_score": 7}', '{"overall_score": 3}']
    v = V.OpenAIShapedVerifier(FakeOpenAI(), "rubric")
    r = V.OpenAIShapedReflector(FakeOpenAI(), "REFLEX", "REFINE")
    refine_kws = (dict(images=images, evaluations=evals, current_prompt=cur, reflections=refl),
                  dict(images=images, current_prompt=cur, reflections=refl),          # nvila branch: no evaluations
                  dict(images=images, evaluations=evals, current_prompt=cur),        # noise + prompt search: no reflections
                  dict())

    def reference_payloads():
        path = ref_path("tts/verifiers/openai_verifier.py")
        ns = {"Union": Union, "Image": Image, "base64": base64, "BytesIO": BytesIO}
        want = {"prepare_inputs", "prepare_refine_prompt_inputs", "prepare_reflexion_prompt_inputs"}
        for node in ast.parse(open(path).read()).body:
            if isinstance(node, ast.ClassDef) and node.name == "OpenAIVerifier":
                for m in node.body:
                    if isinstance(m, ast.FunctionDef) and m.name in want:
                        exec(compile(ast.Module([m], []), path, "exec"), ns)
        assert want <= set(ns)
        return {"inputs": ns["prepare_inputs"](None, images, orig),
                "reflexion": ns["prepare_reflexion_prompt_inputs"](None, images, orig, cur, refl, evals),
                "refine": [ns["prepare_refine_prompt_inputs"](None, orig, **kw) for kw in refine_kws]}

    ref = Store("verifier_adapters").value("message_builders", reference_payloads)
    assert norm(v.prepare_inputs(images, orig)) == ref["inputs"]
    assert norm(r.prepare_reflexion_prompt_inputs(images, orig, cur, refl, evals)) == ref["reflexion"]
    assert norm([r.prepare_refine_prompt_inputs(orig, **kw) for kw in refine_kws]) == ref["refine"]


def test_reflection_generator_messages_equal_the_reference_function():
    """tts_reflectionflow.py:27-41 (the reference function's messages are stored, tests/_refgold.py)"""
    import ast
    from tests._refgold import Store, norm, ref_path
    cases = (("out/00001/midimg/2_round@17.png", 'a "quoted" prompt'), ("data:image/jpeg;base64,AAAA", "x"))

    def reference_messages():
        path = ref_path("tts/tts_reflectionflow.py")
        ns = {}
        for node in ast.parse(open(path).read()).body:
            if isinstance(node, ast.FunctionDef) and node.name == "generate_messages":
                exec(compile(ast.Module([node], []), path, "exec"), ns)
        return [ns["generate_messages"](img, prompt) for img, prompt in cases]

    ref = Store("verifier_adapters").value("generate_messages", reference_messages)
    assert norm([V.ReflectionGeneratorOurs.generate_messages(img, prompt) for img, prompt in cases]) == ref


def test_image_verifier_adapter_over_the_reference_reward_method():
    """reward_modeling/inference.py:71-76,155-180: the reference's `reward()` and `_norm()` methods, compiled out of
    the class and bound to a fake inferencer (model -> logits, no tokenizer / checkpoint), behind `ImageVerifierOurs`:
    the adapter consumes exactly what the reference method returns, batch by batch, and ranks by `Overall` descending.
    What the reference method returned for each batch is stored (tests/_refgold.py) and replayed to the adapter."""
    import ast
    from tests._refgold import Store, norm, ref_path
    batches = []

    class RecordingInferencer:  # the reference's methods bound to a fake model, run while recording
        inference_config = {"VQ_mean": 2.0, "VQ_std": 4.0}

        def __init__(self):
            ns = {}
            for node in ast.parse(open(ref_path("reward_modeling/inference.py")).read()).body:
                if isinstance(node, ast.ClassDef):
                    for m in node.body:
                        if isinstance(m, ast.FunctionDef) and m.name in ("reward", "_norm"):
                            exec(compile(ast.Module([m], []), ref_path("reward_modeling/inference.py"), "exec"), ns)
            assert {"reward", "_norm"} <= set(ns)
            self._reward, self._norm_fn = ns["reward"], ns["_norm"]
            self.calls = []

        def _norm(self, *a, **k):
            return self._norm_fn(self, *a, **k)

        def reward(self, image_paths, prompts, **kw):
            out = self._reward(self, image_paths, prompts, **kw)
            self.calls.append({"n": len(image_paths), "kw": kw, "out": out})
            return out

        def prepare_batch(self, image_paths, prompts, max_pixels):
            return {"pix": [im.getpixel((0, 0))[0] for im in image_paths]}

        def model(self, return_dict, pix):
            return {"logits": torch.tensor([[float(p)] for p in pix])}

    cands = [_cand(i, (10 * i % 256, 0, 0)) for i in (5, 1, 9, 3, 7)]

    def reference_calls():
        inf = RecordingInferencer()
        V.ImageVerifierOurs(inf, batch_size=2).score(cands, ["p"] * 5)
        return inf.calls

    calls = Store("verifier_adapters").value("image_verifier_reward", reference_calls)

    class Inferencer:  # replays what the reference reward() returned, batch by batch
        def reward(self, image_paths, prompts, **kw):
            c = calls[len(batches)]
            batches.append(len(image_paths))
            assert c["n"] == len(image_paths) and c["kw"] == norm(kw)
            return c["out"]

    v = V.ImageVerifierOurs(Inferencer(), batch_size=2)
    out = v.score(cands, ["p"] * 5)
    assert batches == [2, 2, 1]
    assert [o["Overall"] for o in out] == [(10 * i - 2.0) / 4.0 for i in (5, 1, 9, 3, 7)]
    assert all(o["VQ"] == o["Overall"] for o in out)
    ranked = S.sort_outputs(out, "ours", "Overall")
    assert [o["image_name"] for o in ranked] == [cands[k].name for k in (2, 4, 0, 3, 1)]
