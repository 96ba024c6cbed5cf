"""not-gpu: the best-of-N filter over a finished run (reflectionflow_b200/tts/verifier_filter.py, mirror of
tts/verifier_filter.py): candidate order, the yes/no key, bucket folders."""
import json
import os
import sys

import pytest
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from reflectionflow_b200.tts import verifier_filter as VF  # noqa: E402
from reflectionflow_b200.tts.dist import DistCtx  # noqa: E402
from reflectionflow_b200.tts.verifiers import StubVerifier  # noqa: E402


def _make_run(root, rounds=(1, 2, 10), per_round=3):
    folder = os.path.join(root, "00000")
    mid = os.path.join(folder, "midimg")
    os.makedirs(mid)
    with open(os.path.join(folder, "metadata.jsonl"), "w") as f:
        json.dump({"prompt": "a photo of a bench", "tag": "single_object"}, f)
    g = torch.Generator().manual_seed(0)
    names = []
    for r in rounds:
        for k in range(per_round):
            seed = int(torch.randint(0, 2 ** 31 - 1, (1,), generator=g))
            stem = os.path.join(mid, f"{r}_round@{seed}")
            torch.save(torch.randn(1, 16, 64, generator=g).to(torch.bfloat16), stem + ".latent.pt")
            Image.new("RGB", (8, 8), (r * 20 % 256, k * 40, 7)).save(stem + ".png")
            names.append(stem)
    return folder, names


def test_order_key_and_buckets(tmp_path):
    folder, _ = _make_run(str(tmp_path))
    stems = VF.list_candidates(folder)
    rounds = [int(os.path.basename(s).split("_round@")[0]) for s in stems]
    assert rounds == sorted(rounds) and rounds[-1] == 10 and len(stems) == 9     # numeric round order (:75)
    for r in (1, 2, 10):                                                          # name order inside a round (:66)
        part = [os.path.basename(s) for s in stems if os.path.basename(s).startswith(f"{r}_round@")]
        assert part == sorted(part, key=lambda s: s + ".png")
    ver = StubVerifier("nvila")
    res = VF.filter_folder(folder, "a photo of a bench", ver, ctx=DistCtx())
    outs = res["outputs"]
    assert [o["image_name"] for o in outs] == [s + ".png" for s in stems]
    key = lambda o: (0, -o["score"]) if o["label"] == "yes" else (1, o["score"])   # verifier_filter.py:119-123
    for n in VF.BUCKETS:
        want = min(range(min(n, 9)), key=lambda i: (key(outs[i]), i))
        assert res["chosen"][n] == stems[want]
        d = os.path.join(folder, f"nfe{n}")
        assert sorted(os.listdir(d)) == ["00000.latent.pt", "00000.png"]
        assert open(os.path.join(d, "00000.png"), "rb").read() == open(stems[want] + ".png", "rb").read()
    assert res["chosen"][1] == stems[0]            # best of the first one is the first one
    assert res["chosen"][16] == res["chosen"][32]  # fewer than 16 candidates: both buckets see all nine


def test_pixel_verifiers_get_the_stored_png(tmp_path):
    folder, _ = _make_run(str(tmp_path), rounds=(1,), per_round=2)

    class NeedsPixels(StubVerifier):
        needs_images = True

        def value(self, cand):
            assert cand.pil() is not None and cand.pil().size == (8, 8)
            return cand.pil().getpixel((0, 0))[1] / 255.0 - 0.05

    res = VF.filter_folder(folder, "p", NeedsPixels("nvila"), ctx=DistCtx(), buckets=(1, 2))
    stems = VF.list_candidates(folder)
    green = [Image.open(s + ".png").getpixel((0, 0))[1] for s in stems]      # 0 and 40, in name order
    assert [o["label"] for o in res["outputs"]] == ["yes" if gch else "no" for gch in green]
    assert res["chosen"][1] == stems[0] and res["chosen"][2] == stems[green.index(40)]


def test_main_walks_every_prompt_folder(tmp_path):
    run = tmp_path / "run"
    for i in range(2):
        f, _ = _make_run(str(tmp_path / f"tmp{i}"), rounds=(1, 2), per_round=2)
        os.makedirs(run, exist_ok=True)
        os.rename(f, run / f"{i:05}")
    cfg = {"pipeline_args": {"height": 64, "width": 64}, "verifier_args": {"name": "openai"}}
    (tmp_path / "cfg.json").write_text(json.dumps(cfg))
    assert VF.main(["--pipeline_config_path", str(tmp_path / "cfg.json"), "--imgpath", str(run), "--synthetic"],
                   ctx=DistCtx()) == 0
    for i in range(2):
        assert all(os.path.exists(run / f"{i:05}" / f"nfe{n}" / "00000.png") for n in VF.BUCKETS)
    with pytest.raises(RuntimeError, match="no candidates"):
        os.makedirs(run / "00002" / "midimg")
        VF.filter_folder(str(run / "00002"), "p", StubVerifier("nvila"))


def test_filter_equals_the_reference_main(tmp_path):
    """tts/verifier_filter.py::main (:28-176), unmodified, compiled out of its file and run over fakes (argument
    parser, NVILA loader, `Image.open(...).save(...)` recording paths) on the same run directory: the image copied
    into every nfe<N> folder is the same (the reference's choices are stored, tests/_refgold.py)."""
    import ast
    import hashlib
    import types

    import numpy as np
    from tests._refgold import Store, ref_path
    run = tmp_path / "run"
    for i in range(2):
        f, _ = _make_run(str(tmp_path / f"tmp{i}"), rounds=(1, 2, 3, 10), per_round=5)   # 20 candidates: nfe32 = all
        os.makedirs(run, exist_ok=True)
        os.rename(f, run / f"{i:05}")
    cfg = {"pipeline_args": {"height": 64, "width": 64},
           "verifier_args": {"name": "nvila", "model_name": "m", "cache_dir": "c"}}
    (tmp_path / "cfg.json").write_text(json.dumps(cfg))

    def verdict(path):
        v = int(hashlib.sha256(os.path.basename(path).encode()).hexdigest()[:8], 16)
        return ("yes" if v % 4 else "no"), float(np.float32(0.5 + (v % 50) / 100.0))   # coarse scores: ties

    saves = []

    class Opened:
        def __init__(self, path):
            self.path = path

        def save(self, dest):
            saves.append((dest, self.path))

    class ImageMod:
        open = staticmethod(Opened)

    class Nvila:
        @staticmethod
        def generate_content(parts):
            label, score = verdict(parts[0].path)
            logits = torch.zeros(1, 2)
            logits[0, 0 if label == "yes" else 1] = score
            return label, (logits,)

    def reference_choices():
        path = ref_path("tts/verifier_filter.py")
        args = types.SimpleNamespace(pipeline_config_path=str(tmp_path / "cfg.json"), imgpath=str(run), start_index=0,
                                     end_index=-1)
        ns = dict(torch=torch, json=json, os=os, time=__import__("time"), Image=ImageMod, tqdm=lambda it, **kw: it,
                  parse_cli_args=lambda: args, load_model=lambda model_name, cache_dir: (Nvila, 0, 1))
        fn = next(n for n in ast.parse(open(path).read()).body if isinstance(n, ast.FunctionDef) and n.name == "main")
        exec(compile(ast.Module([fn], []), path, "exec"), ns)
        ns["main"]()
        return {os.path.basename(os.path.dirname(os.path.dirname(d))) + "/" + os.path.basename(os.path.dirname(d)):
                os.path.relpath(s, run) for d, s in saves}

    ref_choice = Store("verifier_filter").value("main", reference_choices)

    class Ours(StubVerifier):
        def score_one(self, cand, prompt):
            label, score = verdict(cand.name)
            return {"image_name": cand.name, "label": label, "score": score}

    for i in range(2):
        res = VF.filter_folder(str(run / f"{i:05}"), "a photo of a bench", Ours("nvila"), ctx=DistCtx())
        for n in VF.BUCKETS:
            assert os.path.relpath(res["chosen"][n] + ".png", run) == ref_choice[f"{i:05}/nfe{n}"], (i, n)
