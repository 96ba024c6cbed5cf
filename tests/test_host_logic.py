"""not-gpu: host-side mirror of the reference interface — scheduler, noise factory, pipeline
argument handling, config/CLI schema — checked against the oracle (no kernels involved)."""
import json
import os

import pytest
import torch

from oracle import flux_oracle as fo
from reflectionflow_b200.pipeline import B200FluxPipeline, Condition, flow_match_schedule, generate
from reflectionflow_b200.scheduler import FlowMatchEulerDiscreteScheduler, calculate_shift
from reflectionflow_b200.tts import utils as U


class _Cfg(dict):
    __getattr__ = dict.__getitem__


class FakeTransformer:
    """Records what the pipeline hands to the device loop (test-only; not a compute fallback)."""
    device = torch.device("cpu")
    config = _Cfg(in_channels=64, guidance_embeds=True)

    def __init__(self):
        self.calls = []

    def denoise(self, latents, prompt_embeds, pooled, t_in, sigmas, guidance_scale, img_ids, txt_ids,
                cond_latents=None, cond_ids=None, model_config=None, condition_scale=1.0):
        self.calls.append(dict(latents=latents, t_in=t_in, sigmas=sigmas, g=guidance_scale,
                               img_ids=img_ids, txt_ids=txt_ids, cond=cond_latents, cond_ids=cond_ids,
                               mc=model_config, cs=condition_scale))
        return latents


@pytest.mark.parametrize("steps,seq", [(28, 4096), (4, 256), (50, 4096), (30, 1024)])
def test_schedule_bit_identical_to_oracle(steps, seq):
    ts, sig = flow_match_schedule(steps, seq)
    ots, osig = fo.flow_match_sigmas(steps, seq)
    assert torch.equal(ts, ots) and torch.equal(sig, osig)
    assert calculate_shift(seq) == fo.calculate_shift(seq)


def test_scheduler_object_surface():
    s = FlowMatchEulerDiscreteScheduler()
    assert s.order == 1 and s.config.base_image_seq_len == 256 and s.config.max_shift == 1.15
    s.set_timesteps(sigmas=[1.0, 0.5], mu=0.5)
    assert len(s.timesteps) == 2 and len(s.sigmas) == 3 and s.sigmas[-1] == 0


def test_get_noises_matches_oracle_protocol():
    torch.manual_seed(99)
    a = U.get_noises(2 ** 31 - 1, 4, 256, 256)
    torch.manual_seed(99)
    b = fo.get_noises(2 ** 31 - 1, 4, 256, 256)
    assert list(a) == list(b)
    for k in a:
        assert a[k].dtype == torch.bfloat16 and a[k].shape == (1, 256, 64) and torch.equal(a[k], b[k])
    # side effect kept: the global RNG is left re-seeded with the last seed (SURVEY App. B.5)
    nxt = torch.randint(0, 2 ** 31 - 1, (1,))
    torch.manual_seed(list(a)[-1])
    torch.randn((1, 16, 32, 32), dtype=torch.bfloat16)
    assert torch.equal(nxt, torch.randint(0, 2 ** 31 - 1, (1,)))


def test_pipeline_call_entry_a_hands_reference_timesteps_to_the_loop():
    ft = FakeTransformer()
    pipe = B200FluxPipeline(ft)
    emb, pooled = torch.randn(2, 512, 4096), torch.randn(2, 768)
    lat = torch.randn(2, 4096, 64).to(torch.bfloat16)
    out = pipe(prompt_embeds=emb, pooled_prompt_embeds=pooled, latents=lat, guidance_scale=3.5,
               num_inference_steps=28, height=1024, width=1024, output_type="latent")
    assert out.images.shape == (2, 4096, 64)
    c = ft.calls[0]
    ts, sig = fo.flow_match_sigmas(28, 4096)
    assert torch.equal(c["t_in"], ts.to(torch.bfloat16) / 1000) and torch.equal(c["sigmas"], sig)
    assert c["img_ids"].shape == (4096, 3) and c["txt_ids"].shape == (512, 3) and c["cond"] is None
    assert torch.equal(c["img_ids"].float(), fo.prepare_latent_image_ids(64, 64).float())


def test_pipeline_errors_match_diffusers_semantics():
    pipe = B200FluxPipeline(FakeTransformer())
    e, p = torch.randn(1, 512, 4096), torch.randn(1, 768)
    with pytest.raises(ValueError):
        pipe(prompt_embeds=e, pooled_prompt_embeds=p, height=1000, width=1024, output_type="latent")
    with pytest.raises(ValueError):
        pipe(prompt="x", prompt_embeds=e, pooled_prompt_embeds=p, output_type="latent")
    with pytest.raises(ValueError):
        pipe(output_type="latent")
    with pytest.raises(ValueError):
        pipe(prompt_embeds=e, output_type="latent")
    with pytest.raises(NotImplementedError):  # no text encoders attached
        pipe(prompt="a cat", output_type="latent")
    with pytest.raises(NotImplementedError):  # no VAE attached
        pipe(prompt_embeds=e, pooled_prompt_embeds=p, height=64, width=64)


def test_generate_entry_b_condition_ids_and_defaults():
    ft = FakeTransformer()
    pipe = B200FluxPipeline(ft)
    e, p = torch.randn(1, 512, 4096), torch.randn(1, 768)
    cond_lat = torch.randn(1, 1024, 64)
    cond = Condition("cot", latents=cond_lat, position_delta=[0, -32])
    out = generate(pipe, conditions=[cond], model_config={"union_cond_attn": True}, default_lora=True,
                   prompt_embeds=e, pooled_prompt_embeds=p, height=1024, width=1024,
                   output_type="latent")
    c = ft.calls[0]
    assert out.images.shape == (1, 4096, 64)
    assert c["t_in"].numel() == 28 and c["g"] == 3.5  # defaults of generate.py:30,32
    assert c["cond"].shape == (1, 1024, 64)
    assert torch.equal(c["cond_ids"].float(), fo.condition_ids(512, (0, -32)).float())
    with pytest.raises(AssertionError):
        generate(pipe, conditions=[cond, cond], prompt_embeds=e, pooled_prompt_embeds=p,
                 output_type="latent")
    with pytest.raises(NotImplementedError):
        Condition("no_such_type", latents=cond_lat)
    assert Condition("depth", latents=cond_lat).type_id == 0  # every type of condition.py:10-21 runs the same path
    # defaults: 512 x 512 like generate.py:28-29
    generate(pipe, conditions=None, prompt_embeds=e, pooled_prompt_embeds=p, output_type="latent")
    assert ft.calls[-1]["latents"].shape == (1, 1024, 64) and ft.calls[-1]["cond"] is None


def test_prepare_latents_cpu_generator_protocol():
    pipe = B200FluxPipeline(FakeTransformer())
    g = torch.Generator().manual_seed(5)
    lat, ids = pipe.prepare_latents(1, 16, 256, 256, torch.bfloat16, "cpu", g)
    g2 = torch.Generator().manual_seed(5)
    ref = fo.pack_latents(torch.randn((1, 16, 32, 32), generator=g2, dtype=torch.bfloat16), 1, 16, 32, 32)
    assert torch.equal(lat, ref) and ids.shape == (256, 3)


def test_config_schema_and_cli():
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = json.load(open(os.path.join(here, "reflectionflow_b200", "tts", "configs",
                                      "headline_tree_flux_dev.json")))
    for sec in ("pipeline_args", "verifier_args", "refine_args", "search_args", "model",
                "reflection_args", "prompt_refiner_args", "use_low_gpu_vram", "batch_size_for_img_gen"):
        assert sec in cfg
    assert set(cfg["model"]) == {"add_cond_attn", "latent_lora", "union_cond_attn"}
    # same schema as the reference's shipped config (a copy is stored under tests/golden/)
    ref_cfg = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_configs", "flux.1_dev_nvilascore.json")
    r = json.load(open(ref_cfg))
    assert set(r) == set(cfg)
    for k in r:
        if isinstance(r[k], dict):
            assert set(r[k]) == set(cfg[k]), k
    a = U.parse_cli_args(["--pipeline_config_path", "x.json", "--start_index", "3", "--imgpath", "d"])
    assert a.pipeline_config_path == "x.json" and a.start_index == 3 and a.end_index == -1
    assert a.output_dir == "output" and a.meta_path == "meta.jsonl" and a.imgpath == "d"
    assert U.TORCH_DTYPE_MAP["bf16"] is torch.bfloat16
    with pytest.raises(KeyError):
        U.get_latent_prep_fn("stabilityai/stable-diffusion-xl-base-1.0")


def test_t5_bucket_table_matches_transformers():
    """host-side relative-position buckets of the native T5 encoder (text.py) vs transformers'"""
    import torch
    from transformers.models.t5.modeling_t5 import T5Attention
    from reflectionflow_b200.text import t5_bucket_table
    for seq in (1, 7, 77, 128, 512):
        pos = torch.arange(seq)
        rel = pos[None, :] - pos[:, None]
        ref = T5Attention._relative_position_bucket(rel, bidirectional=True, num_buckets=32, max_distance=128)
        assert torch.equal(t5_bucket_table(seq), ref), seq


def test_byte_tokenizer_shapes_and_eos():
    import torch
    from reflectionflow_b200.tts.verifiers import ByteTokenizer
    clip = ByteTokenizer(49408, eos=49407, pad=49407, bos=49406)
    ids = clip(["a cat", "x" * 200], 77)
    assert ids.shape == (2, 77) and ids.dtype == torch.long
    assert ids[0, 0] == 49406 and ids[0, 6] == 49407 and (ids[0, 6:] == 49407).all()
    assert ids[1, -1] == 49407 and ids.max() < 49408 and ids.min() >= 0
    assert int(ids[0].argmax()) == 6           # CLIP pools at the first EOS (largest id)
    t5 = ByteTokenizer(32128, eos=1, pad=0)
    ids = t5(["hello"], 512)
    assert ids.shape == (1, 512) and ids[0, 5] == 1 and (ids[0, 6:] == 0).all()


def test_artefact_saver_orders_writes_per_path_and_flushes(tmp_path):
    """tts.reflectionflow: artefact writes run on a thread pool; two writes to the same path keep their
    submission order, flush_saves() joins everything and re-raises a failed write."""
    import time
    from reflectionflow_b200.tts import reflectionflow as RF
    p = str(tmp_path / "a.bin")
    order = []

    def slow():
        time.sleep(0.2)
        order.append("first")
        open(p, "wb").write(b"first")

    def fast():
        order.append("second")
        open(p, "wb").write(b"second")
    RF._submit_save(p, slow)
    RF._submit_save(p, fast)
    for i in range(16):  # other paths run concurrently
        q = str(tmp_path / f"f{i}.bin")
        RF._submit_save(q, lambda q=q: open(q, "wb").write(b"x"))
    RF.flush_saves()
    assert order == ["first", "second"] and open(p, "rb").read() == b"second"
    assert len(os.listdir(tmp_path)) == 17

    def boom():
        raise OSError("disk full")
    RF._submit_save(str(tmp_path / "bad"), boom)
    with pytest.raises(OSError):
        RF.flush_saves()
    RF.flush_saves()  # the failed future was consumed


def test_candidate_png_is_encoded_once():
    import numpy as np
    from PIL import Image
    from reflectionflow_b200.tts.verifiers import Candidate
    img = Image.fromarray((np.arange(64 * 64 * 3) % 251).astype("uint8").reshape(64, 64, 3))
    c = Candidate("x/1_round@7.png", 7, image=img)
    b1 = c.png_bytes()
    assert b1 is c.png_bytes() and b1[:8] == b"\x89PNG\r\n\x1a\n"
    import io
    assert np.array_equal(np.asarray(Image.open(io.BytesIO(b1))), np.asarray(img))
    assert Candidate("y", 0).png_bytes() is None


def test_bench_accounting_matches_the_survey():
    """bench.py's work counts are the ones SURVEY.md §8(d) / BASELINE.md quote (the judge recomputes TFLOP/s from
    them): 57 (24 D^2 N + 4 N^2 D), entry A N = 4608 -> 74.385 TFLOP, entry B N = 5632 -> 94.954 TFLOP; and the
    roofline denominator comes from the driver-written MEASURED_PEAKS.json when it is there."""
    import importlib.util, json, os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("rf_bench", os.path.join(root, "bench.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    assert (b.N_TXT, b.N_IMG, b.N_COND) == (512, 4096, 1024)
    assert abs(b.algorithmic_tflop(4608) - 74.385) < 0.05
    assert abs(b.algorithmic_tflop(5632) - 94.954) < 0.05
    assert abs(b.algorithmic_tflop(768) - 10.348) < 0.03  # the survey adds ~0.02 TFLOP of embedders / modulation
    pk = b.peaks()
    mp = os.path.join(root, "MEASURED_PEAKS.json")
    if os.path.exists(mp):
        m = json.load(open(mp))
        assert pk["tflops_sustained"] == m["bf16_tflops_sustained"] and "measured" in pk["source"]
    assert b.physical_cores() >= 1


def test_get_config_follows_the_reference(tmp_path, monkeypatch):
    """generate.py:16-22: explicit path, else $XFL_CONFIG, else {} ; generate() takes model_config from its "model" key"""
    from reflectionflow_b200.pipeline import get_config, seed_everything
    monkeypatch.delenv("XFL_CONFIG", raising=False)
    assert get_config() == {}
    y = tmp_path / "c.yaml"
    y.write_text("model:\n  union_cond_attn: true\n  add_cond_attn: false\ntrain:\n  lr: 1\n")
    assert get_config(str(y))["model"] == {"union_cond_attn": True, "add_cond_attn": False}
    monkeypatch.setenv("XFL_CONFIG", str(y))
    assert get_config()["train"] == {"lr": 1}
    seed_everything(7)
    a = torch.rand(3)
    seed_everything(7)
    assert torch.equal(a, torch.rand(3))


def test_image_helpers_of_tts_utils(tmp_path):
    """tts/utils.py:188-208"""
    import io
    from PIL import Image
    from reflectionflow_b200.tts.utils import convert_to_bytes, load_image
    im = Image.new("RGBA", (5, 3), (10, 20, 30, 40))
    assert load_image(im) is im
    p = tmp_path / "x.png"
    im.save(p)
    assert load_image(str(p)).size == (5, 3)
    back = Image.open(io.BytesIO(convert_to_bytes(str(p))))
    assert back.mode == "RGB" and back.format == "PNG" and back.getpixel((0, 0)) == (10, 20, 30)
    assert convert_to_bytes(im) == convert_to_bytes(str(p))


def test_pipeline_tools_module_level_forms():
    """pipeline_tools.py:7-52: `encode_images(pipeline, images)` and `prepare_text_input(pipeline, prompts, ...)` keep
    the reference's call shape and hand the reference's fixed arguments to the pipeline"""
    from reflectionflow_b200 import pipeline as P
    seen = {}

    class Pipe:
        device = "cpu"

        def encode_images(self, images, eps=None, generator=None):
            seen["img"] = (images, eps, generator)
            return "tokens", "ids"

        def encode_prompt(self, **kw):
            seen["txt"] = kw
            return "pe", "pooled", "text_ids"

    assert P.encode_images(Pipe(), "IMG") == ("tokens", "ids") and seen["img"] == ("IMG", None, None)
    assert P.prepare_text_input(Pipe(), ["a", "b"], max_sequence_length=256) == ("pe", "pooled", "text_ids")
    assert seen["txt"] == dict(prompt=["a", "b"], prompt_2=None, prompt_embeds=None, pooled_prompt_embeds=None,
                               device="cpu", num_images_per_prompt=1, max_sequence_length=256, lora_scale=None)


def _reference_functions(relpath, names, extra=None):
    """the named top-level functions of a reference file, compiled in isolation (the module itself imports packages
    that are not installed); run only while recording the stored reference results (tests/_refgold.py)"""
    import ast
    from tests._refgold import ref_path
    path = ref_path(relpath)
    ns = dict(extra or {})
    for node in ast.parse(open(path).read()).body:
        if isinstance(node, ast.FunctionDef) and node.name in names:
            exec(compile(ast.Module([node], []), path, "exec"), ns)
    return ns


def test_small_utils_agree_with_the_reference(tmp_path):
    """tts/utils.py:157-222: prompt_to_filename, recover_json_from_output, get_batches, load_verifier_prompt — known
    answers, and what the reference's own functions returned on the same inputs (stored, tests/_refgold.py)"""
    import hashlib, json, re
    from reflectionflow_b200.tts import utils as U
    long_prompt = "A photo of: two cats & a dog!! " * 6
    assert U.prompt_to_filename("a red cube") == "prompt@a_red_cube_hash@" + hashlib.sha256(b"a red cube").hexdigest()[:8]
    # upstream arithmetic: max_length - 8 - 7 prompt characters + "prompt@" + "_hash@" + 8 = max_length + 6
    assert len(U.prompt_to_filename(long_prompt)) == 106 and "__" not in U.prompt_to_filename(long_prompt)
    assert U.recover_json_from_output('noise {"a": {"b": 1}} trailing') == {"a": {"b": 1}}
    assert U.get_batches(list(range(5)), 2) == [[0, 1], [2, 3], [4]]
    (tmp_path / "p.txt").write_text('"""rubric"""\nline')
    (tmp_path / "p.json").write_text('{"position": "grade"}')
    assert U.load_verifier_prompt(str(tmp_path / "p.txt")) == "rubric\nline"
    assert U.load_verifier_prompt(str(tmp_path / "p.json")) == {"position": "grade"}
    with pytest.raises(ValueError):
        U.load_verifier_prompt("x.yaml")
    from tests._refgold import Store, norm
    prompts = ("a red cube", long_prompt, "  ümlaut/слово  ", "")
    outs = ('x {"k": [1, {"z": 2}]} y', '{"only": true}')

    def reference_results():
        ref = _reference_functions("tts/utils.py", {"prompt_to_filename", "recover_json_from_output", "get_batches",
                                                    "load_verifier_prompt"},
                                   {"re": re, "hashlib": hashlib, "json": json})
        return {"prompt_to_filename": [ref["prompt_to_filename"](p) for p in prompts],
                "prompt_to_filename_40": [ref["prompt_to_filename"](p, 40) for p in prompts],
                "recover_json_from_output": [ref["recover_json_from_output"](o) for o in outs],
                "get_batches": [list(ref["get_batches"](list(range(6)), n)) for n in (1, 2, 7)],
                "load_verifier_prompt": [ref["load_verifier_prompt"](str(tmp_path / f)) for f in ("p.txt", "p.json")]}

    ref = Store("host_logic").value("small_utils", reference_results)
    assert [U.prompt_to_filename(p) for p in prompts] == ref["prompt_to_filename"]
    assert [U.prompt_to_filename(p, 40) for p in prompts] == ref["prompt_to_filename_40"]
    assert norm([U.recover_json_from_output(o) for o in outs]) == ref["recover_json_from_output"]
    assert norm([list(U.get_batches(list(range(6)), n)) for n in (1, 2, 7)]) == ref["get_batches"]
    assert norm([U.load_verifier_prompt(str(tmp_path / f)) for f in ("p.txt", "p.json")]) == ref["load_verifier_prompt"]


def test_param_count_is_flux_dev():
    """SURVEY App. A.1: 11.901 B parameters (double block 339.8 M, single 141.6 M)"""
    from reflectionflow_b200.config import FluxDiTConfig
    n = FluxDiTConfig().param_count()
    assert abs(n / 1e9 - 11.901) < 0.005
    one_double = FluxDiTConfig(num_layers=1, num_single_layers=0).param_count() - \
        FluxDiTConfig(num_layers=0, num_single_layers=0).param_count()
    one_single = FluxDiTConfig(num_layers=0, num_single_layers=1).param_count() - \
        FluxDiTConfig(num_layers=0, num_single_layers=0).param_count()
    assert abs(one_double / 1e6 - 339.8) < 0.1 and abs(one_single / 1e6 - 141.6) < 0.1


def test_condition_encode_follows_the_reference_class():
    """train_flux/flux/condition.py:24-132: the reference's Condition class, compiled out of its file, and ours, over
    the same fake `encode_images`: tokens, shifted position ids (`position_delta`, the "subject" default) and the
    type-id column are equal; the type-id table is the reference's."""
    import ast
    from typing import List, Optional, Tuple, Union
    from PIL import Image
    from reflectionflow_b200 import pipeline as P
    import hashlib
    from tests._refgold import Store, ref_path
    path = ref_path("train_flux/flux/condition.py")
    assert P.condition_dict["cot"] == 12 and P.Condition.get_type_id("cot") == 12

    def fake_encode(pipe, image):
        w, h = image.size
        n = (w // 16) * (h // 16)
        g = torch.Generator().manual_seed(w * 1000 + h)
        ids = torch.zeros(n, 3)
        ids[:, 1] = torch.arange(n) // (w // 16)
        ids[:, 2] = torch.arange(n) % (w // 16)
        return torch.randn(1, n, 64, generator=g), ids

    class Pipe:
        device, dtype = "cpu", torch.float32

        def encode_images(self, images, eps=None, generator=None):
            return fake_encode(self, images)

    # raw image -> condition image (condition.py:43-80), for the types that need no network model
    raw = Image.fromarray((torch.rand(48, 80, 3, generator=torch.Generator().manual_seed(2)) * 255).to(torch.uint8).numpy())
    img = Image.new("RGB", (64, 32), (9, 9, 9))
    ctypes_raw = ("canny", "subject", "coloring", "deblurring", "fill", "cartoon")
    encodes = (("cot", [0, -2]), ("cot", None), ("subject", None), ("canny", [3, 1]))

    def image_rec(im):
        return [im.mode, list(im.size), hashlib.sha256(im.tobytes()).hexdigest()]

    def tensors_rec(ts):
        return [[list(t.shape), hashlib.sha256(t.float().contiguous().numpy().tobytes()).hexdigest()] for t in ts]

    def reference_results():
        import cv2  # used by the reference class through its module namespace
        import numpy as np
        from PIL import ImageFilter
        ns = dict(torch=torch, Optional=Optional, Union=Union, List=List, Tuple=Tuple, Image=Image, FluxPipeline=object,
                  encode_images=fake_encode, cv2=cv2, np=np, ImageFilter=ImageFilter)
        for node in ast.parse(open(path).read()).body:
            if isinstance(node, ast.ClassDef) and node.name == "Condition" or \
                    isinstance(node, ast.Assign) and getattr(node.targets[0], "id", "") == "condition_dict":
                exec(compile(ast.Module([node], []), path, "exec"), ns)
        C = ns["Condition"]
        return {"condition_dict": ns["condition_dict"],
                "raw": [image_rec(C(condition_type=t, raw_img=raw).condition) for t in ctypes_raw],
                "encode": [tensors_rec(C(condition_type=t, condition=img, position_delta=d).encode(Pipe()))
                           for t, d in encodes]}

    ref = Store("host_logic").value("condition", reference_results)
    assert ref["condition_dict"] == P.condition_dict
    # raw image -> condition image (condition.py:43-80), for the types that need no network model
    for ctype, want in zip(ctypes_raw, ref["raw"]):
        assert image_rec(P.Condition(ctype, raw_img=raw).condition) == want, ctype
    with pytest.raises(NotImplementedError):
        P.Condition("depth", raw_img=raw)
    for (ctype, delta), want in zip(encodes, ref["encode"]):
        assert tensors_rec(P.Condition(ctype, condition=img, position_delta=delta).encode(Pipe())) == want, (ctype, delta)


def test_tranformer_forward_takes_the_reference_parameter_names():
    """transformer.py:18-44 `prepare_params`: every keyword the reference accepts is either consumed or refused loudly"""
    import ast
    import inspect
    from reflectionflow_b200 import transformer as T
    calls = []

    class Fake:
        condition_scale = 1.0

        def _forward(self, *a):
            calls.append(a)
            return torch.zeros(1, 4, 64)

    kw = dict(hidden_states=torch.zeros(1, 4, 64), encoder_hidden_states=1, pooled_projections=2, timestep=3, img_ids=4,
              txt_ids=5, guidance=6, joint_attention_kwargs=None, controlnet_block_samples=None,
              controlnet_single_block_samples=None)
    out = T.tranformer_forward(Fake(), "cl", "ci", None, {"union_cond_attn": True}, 0, return_dict=False, **kw)
    assert isinstance(out, tuple) and calls[0][1:7] == (1, 2, 3, 4, 5, 6) and calls[0][7:9] == ("cl", "ci")
    assert hasattr(T.tranformer_forward(Fake(), None, None, None, **kw), "sample")
    for bad in (dict(controlnet_block_samples=[0]), dict(controlnet_single_block_samples=[0]),
                dict(joint_attention_kwargs={"scale": 0.5})):
        with pytest.raises(NotImplementedError):
            T.tranformer_forward(Fake(), None, None, None, **dict(kw, **bad))
    with pytest.raises(NotImplementedError):
        T.tranformer_forward(Fake(), None, None, None, {}, 1, **kw)
    from tests._refgold import Store, ref_path

    def reference_names():
        from typing import Any, Dict, Optional
        path = ref_path("train_flux/flux/transformer.py")
        ns = dict(torch=torch, Optional=Optional, Dict=Dict, Any=Any)
        fn = next(n for n in ast.parse(open(path).read()).body
                  if isinstance(n, ast.FunctionDef) and n.name == "prepare_params")
        exec(compile(ast.Module([fn], []), path, "exec"), ns)
        return [p for p in inspect.signature(ns["prepare_params"]).parameters if p != "kwargs"]

    names = Store("host_logic").value("prepare_params", reference_names)
    assert set(names) == set(kw) | {"return_dict"}
