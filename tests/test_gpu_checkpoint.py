"""-m gpu: `B200FluxPipeline.from_pretrained` on a diffusers-layout checkpoint written by
tools/make_synthetic_checkpoint.py at full width and reduced depth (1 double + 2 single blocks, 2 T5 and 2 CLIP
layers).  Loading from disk must compute exactly what the existing state-dict path computes on the same tensors,
whatever the storage (one or three shards, bf16 or fp32, plain directory or hub cache); the text encoders must
match transformers through the checkpoint's own tokenizers; the device staging stays near two tensors; and the
ReflectionFlow script runs on the checkpoint without --synthetic."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from reflectionflow_b200 import _lib as L  # noqa: E402
from reflectionflow_b200 import checkpoint as ck  # noqa: E402
from reflectionflow_b200.pipeline import B200FluxPipeline, Condition, generate  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_synthetic_checkpoint",
                                               os.path.join(ROOT, "tools", "make_synthetic_checkpoint.py"))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)

DEPTH = dict(layers=(1, 2), t5_layers=2, clip_layers=2, width="full")
LORA_RANK = 16
PROMPTS = ["a photo of a red cube on a blue sphere", "two dogs next to a large yellow house"]
H = W = 256


@pytest.fixture(scope="module")
def ckpt(tmp_path_factory):
    base = tmp_path_factory.mktemp("gpu_ckpt")
    dirs = {"one": mk.write_checkpoint(str(base / "one"), shards=1, device="cuda", **DEPTH),
            "three": mk.write_checkpoint(str(base / "three"), shards=3, device="cuda", **DEPTH),
            "fp32": mk.write_checkpoint(str(base / "fp32"), shards=2, dtype="fp32", device="cuda", **DEPTH)}
    # the hub cache layout: refs/main names a snapshot (a link to the files, as the hub's blob links are)
    repo = base / "hub" / "models--black-forest-labs--FLUX.1-dev"
    os.makedirs(repo / "refs")
    os.makedirs(repo / "snapshots")
    (repo / "refs" / "main").write_text(mk.REVISION)
    os.symlink(dirs["one"], repo / "snapshots" / mk.REVISION)
    dirs["hub"] = str(base / "hub")
    dirs["lora"] = mk.write_lora(str(base / "lora"), DEPTH["layers"], "full", rank=LORA_RANK)
    return dirs


def _noise(seed, n=1):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, (H // 16) * (W // 16), 64, generator=g).to(torch.bfloat16).cuda()


def _outputs(pipe):
    """entry B (a Condition image encoded by the VAE, LoRA on) and entry A (a batch of two prompts), as latents
    and as uint8 pixels."""
    img = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (128, 128, 3), dtype=np.uint8))
    eps = torch.randn(16, 16, 16, generator=torch.Generator().manual_seed(3)).to(torch.bfloat16)
    out = {}
    for ot in ("latent", "u8"):
        cond = Condition("cot", condition=img, position_delta=[0, -8], eps=eps)
        out["B/" + ot] = generate(pipe, prompt=[PROMPTS[0]], conditions=[cond], height=H, width=W,
                                  num_inference_steps=2, latents=_noise(1), output_type=ot, default_lora=True,
                                  model_config={"union_cond_attn": True}).images.clone()
        out["A/" + ot] = pipe(prompt=PROMPTS, height=H, width=W, num_inference_steps=2, max_sequence_length=128,
                              latents=_noise(2, 2), output_type=ot).images.clone()
    torch.cuda.synchronize()
    return out


def _close(pipe):
    for m in (pipe.transformer, pipe.vae, getattr(pipe, "text_encoders", None)):
        if m is not None:
            m.close()


def _same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), k


def _state(component_dir):
    from safetensors.torch import load_file
    sd = {}
    for f in sorted(set(ck.weight_files(component_dir).values())):
        sd.update(load_file(f))
    return sd


@pytest.fixture(scope="module")
def reference_outputs(ckpt):
    pipe = B200FluxPipeline.from_pretrained(ckpt["one"], lora_rank=LORA_RANK)
    pipe.load_lora_weights(ckpt["lora"])
    out = _outputs(pipe)
    _close(pipe)
    return out


def test_from_pretrained_equals_the_state_dict_path(ckpt, reference_outputs):
    """The same tensors through from_state_dict / load_state_dict / load_t5_state_dict / load_clip_state_dict and
    the same tokenizer ids give bit-identical outputs."""
    from reflectionflow_b200.scheduler import FlowMatchEulerDiscreteScheduler
    from reflectionflow_b200.text import B200TextEncoders
    from reflectionflow_b200.vae import B200AutoencoderKL
    root = ckpt["one"]
    cfg = lambda c, n="config.json": ck.read_json(os.path.join(root, c, n))  # noqa: E731
    pipe = B200FluxPipeline.from_state_dict(_state(os.path.join(root, "transformer")),
                                            config=ck.dit_config(cfg("transformer")), lora_rank=LORA_RANK)
    pipe.vae = B200AutoencoderKL(**ck.vae_config(cfg("vae"))).load_state_dict(_state(os.path.join(root, "vae")))
    fields, eos = ck.text_config(cfg("text_encoder"), cfg("text_encoder_2"))
    enc = B200TextEncoders(**fields)
    enc.load_t5_state_dict(_state(os.path.join(root, "text_encoder_2")))
    enc.load_clip_state_dict(_state(os.path.join(root, "text_encoder")))
    assert eos == enc.clip_eos_token_id == 2
    pipe.text_encoders = enc
    pipe.text_encoder_hook = enc.as_hook(*ck.tokenizer_fns(root))
    pipe.scheduler = FlowMatchEulerDiscreteScheduler(**ck.scheduler_config(cfg("scheduler", "scheduler_config.json")))
    pipe.load_lora_weights(ckpt["lora"])
    out = _outputs(pipe)
    _close(pipe)
    _same(out, reference_outputs)
    assert out["A/u8"].shape == (2, H, W, 3) and out["A/u8"].dtype == torch.uint8
    assert not torch.equal(out["A/latent"][0], out["A/latent"][1])  # the two prompts differ


@pytest.mark.parametrize("variant", ["three", "fp32", "hub"])
def test_storage_does_not_change_results(ckpt, reference_outputs, variant):
    if variant == "hub":
        pipe = B200FluxPipeline.from_pretrained("black-forest-labs/FLUX.1-dev", cache_dir=ckpt["hub"],
                                                torch_dtype="bf16", lora_rank=LORA_RANK)
    else:
        pipe = B200FluxPipeline.from_pretrained(ckpt[variant], lora_rank=LORA_RANK)
    pipe.load_lora_weights(ckpt["lora"])
    out = _outputs(pipe)
    _close(pipe)
    _same(out, reference_outputs)


def test_staging_memory_is_about_two_tensors(ckpt):
    """torch.cuda.max_memory_allocated counts the staging copies only: the handles allocate with cudaMalloc."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    pipe = B200FluxPipeline.from_pretrained(ckpt["fp32"], lora_rank=LORA_RANK)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    largest = 0
    for comp in ("transformer", "vae", "text_encoder", "text_encoder_2"):
        from safetensors import safe_open
        for k, f in ck.weight_files(os.path.join(ckpt["fp32"], comp)).items():
            with safe_open(f, "pt") as h:
                largest = max(largest, int(np.prod(h.get_slice(k).get_shape())) * 2)  # bf16 bytes on the device
    print(f"staging peak {peak / 2**20:.1f} MiB, largest bf16 tensor {largest / 2**20:.1f} MiB")
    _close(pipe)
    assert peak <= 2 * largest + (16 << 20)


def _hf_text_models(tmp_path):
    """transformers' own save_pretrained of random T5EncoderModel / CLIPTextModel (bf16-representable weights),
    with their fp32 and bf16 CPU models."""
    import copy
    from transformers import CLIPTextConfig, CLIPTextModel, T5Config, T5EncoderModel
    t5cfg = T5Config(vocab_size=32128, d_model=1024, d_kv=64, d_ff=2560, num_layers=2, num_heads=16,
                     feed_forward_proj="gated-gelu", layer_norm_epsilon=1e-6, relative_attention_num_buckets=32,
                     relative_attention_max_distance=128, dropout_rate=0.0)
    clipcfg = CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=2,
                             num_attention_heads=12, max_position_embeddings=77, hidden_act="quick_gelu",
                             eos_token_id=2, bos_token_id=0, pad_token_id=1)
    models = {}
    for name, cls, cfg in (("text_encoder_2", T5EncoderModel, t5cfg), ("text_encoder", CLIPTextModel, clipcfg)):
        cfg._attn_implementation = "eager"
        torch.manual_seed(len(name))
        m32 = cls(cfg).eval()
        with torch.no_grad():
            for n, p in m32.named_parameters():  # unit-variance activations (the HF init is tiny)
                if "layer_norm" in n and n.endswith("weight"):
                    p.copy_(1 + 0.1 * torch.randn_like(p))
                elif n.endswith("bias") and "relative_attention_bias" not in n:
                    p.copy_(0.05 * torch.randn_like(p))
                elif "relative_attention_bias" in n or "shared" in n or "embedding" in n:
                    p.copy_(torch.randn_like(p) * (1.0 if name == "text_encoder_2" else 0.5))
                elif n.endswith(".q.weight") or n.endswith(".k.weight"):
                    p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5 * 0.6)
                else:
                    p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5)
                p.copy_(p.to(torch.bfloat16).float())
        m16 = copy.deepcopy(m32).to(torch.bfloat16)
        m16.save_pretrained(str(tmp_path / name))
        models[name] = (m32, m16)
    return models


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().mean() / b.abs().mean()).item()


def test_text_encoders_from_save_pretrained_match_transformers(ckpt, tmp_path):
    from reflectionflow_b200.text import B200TextEncoders
    models = _hf_text_models(tmp_path)
    enc = B200TextEncoders.from_pretrained(str(tmp_path / "text_encoder"), str(tmp_path / "text_encoder_2"))
    tok, tok2 = ck.tokenizer_fns(ckpt["one"])
    prompts = PROMPTS + [" ".join(["a small green tree and a bright painting of a cat"] * 20)]
    ids, ids2 = tok(prompts, 77), tok2(prompts, 128)
    embeds, pooled = enc.as_hook(tok, tok2)(prompts, None, 128)
    torch.cuda.synchronize()
    with torch.no_grad():
        t5_32, t5_16 = (m(input_ids=ids2)[0] for m in models["text_encoder_2"])
        c32, c16 = (m(input_ids=ids).pooler_output for m in models["text_encoder"])
    e_ref, e_ours = _rel(t5_16, t5_32), _rel(embeds, t5_32)
    p_ref, p_ours = _rel(c16, c32), _rel(pooled, c32)
    print(f"T5 ref-bf16 {e_ref:.3e} ours {e_ours:.3e}; CLIP pooled ref-bf16 {p_ref:.3e} ours {p_ours:.3e}")
    assert embeds.shape == (3, 128, 1024) and pooled.shape == (3, 768)
    assert e_ours <= 1.25 * e_ref + 1e-4
    assert p_ours <= 1.5 * p_ref + 1e-4  # 3 x 768 values: the noisier statistic test_gpu_text.py allows too
    enc.close()


def test_reflectionflow_main_runs_on_the_checkpoint(ckpt, tmp_path, monkeypatch):
    """tts/reflectionflow.py main() without --synthetic: the repo id resolved in the hub cache, the LoRA rank read
    from lora_path, 2 candidates x 1 round x 2 steps, stub verifier and reflector."""
    from PIL import Image
    from reflectionflow_b200.tts import reflectionflow
    from reflectionflow_b200.tts.dist import DistCtx
    from reflectionflow_b200.tts.verifiers import StubReflector, StubVerifier
    seen = {}
    real = B200FluxPipeline.from_pretrained.__func__

    def spy(cls, *a, **k):
        seen.update(k)
        pipe = real(cls, *a, **k)
        seen["pipe"] = pipe
        return pipe
    monkeypatch.setattr(B200FluxPipeline, "from_pretrained", classmethod(spy))
    cfg = {"pipeline_args": {"pretrained_model_name_or_path": "black-forest-labs/FLUX.1-dev",
                             "cache_dir": ckpt["hub"], "torch_dtype": "bf16", "height": H, "width": W,
                             "condition_size": 128, "max_sequence_length": 512, "guidance_scale": 3.5,
                             "num_inference_steps": 2, "lora_path": ckpt["lora"]},
           "verifier_args": {"name": "nvila", "model_name": "stub", "cache_dir": "x"},
           "refine_args": {"name": "openai", "choice_of_metric": "overall_score", "max_new_tokens": 64,
                           "refine_prompt_relpath": "r.txt", "reflexion_prompt_relpath": "x.txt",
                           "verifier_prompt_relpath": "v.json"},
           "search_args": {"search_method": "random", "search_branch": 2, "search_rounds": 1},
           "model": {"add_cond_attn": False, "latent_lora": False, "union_cond_attn": True},
           "reflection_args": {"run_reflection": True, "name": "openai"},
           "prompt_refiner_args": {"run_refinement": True}, "use_low_gpu_vram": False, "batch_size_for_img_gen": 1}
    json.dump(cfg, open(tmp_path / "cfg.json", "w"))
    s0 = tmp_path / "s0" / "00000"
    os.makedirs(s0 / "samples")
    (s0 / "metadata.jsonl").write_text(json.dumps({"prompt": PROMPTS[0], "tag": "position"}) + "\n")
    rng = np.random.default_rng(5)
    for seed in (11, 12):  # round-0 candidates as PNGs
        Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(s0 / "samples" / f"0_round@{seed}.png")

    def two_steps(pipe, **kw):
        return generate(pipe, num_inference_steps=2, **kw)
    rc = reflectionflow.main(["--pipeline_config_path", str(tmp_path / "cfg.json"), "--imgpath", str(tmp_path / "s0"),
                              "--output_dir", str(tmp_path / "s1"), "--seed", "0"], ctx=DistCtx(0, 1, "cuda:0"),
                             verifier=StubVerifier("nvila"), reflector=StubReflector(), generate_fn=two_steps)
    assert rc == 0
    assert seen["lora_rank"] == LORA_RANK and seen["cache_dir"] == ckpt["hub"]
    assert seen["pipe"].transformer.lora_rank == LORA_RANK and seen["pipe"].transformer.has_lora
    out = tmp_path / "s1" / "00000"
    mid = sorted(os.listdir(out / "midimg"))
    assert sum(f.endswith(".png") for f in mid) == 2 and sum(f.endswith(".latent.pt") for f in mid) == 2
    for d in ("samples_lastround", "samples_best", "samples_path_bestround"):
        assert any(f.endswith(".png") for f in os.listdir(out / d)), d
    with Image.open(out / "midimg" / [f for f in mid if f.endswith(".png")][0]) as im:
        assert im.size == (W, H) and im.mode == "RGB"
    _close(seen["pipe"])


def _rewrite(src_dir, dst_dir, edit):
    from safetensors.torch import save_file
    os.makedirs(dst_dir)
    sd = _state(src_dir)
    edit(sd)
    save_file(sd, os.path.join(dst_dir, "diffusion_pytorch_model.safetensors"))
    with open(os.path.join(src_dir, "config.json")) as f, open(os.path.join(dst_dir, "config.json"), "w") as g:
        g.write(f.read())
    return dst_dir


@pytest.mark.parametrize("comp,gone", [
    pytest.param("transformer", "single_transformer_blocks.1.proj_mlp.bias", id="transformer"),
    pytest.param("vae", "decoder.up_blocks.2.resnets.1.conv2.weight", id="vae"),
    # one row slice of the mid-block attention's stacked q | k | v projection
    pytest.param("vae", "decoder.mid_block.attentions.0.to_k.weight", id="vae-mid-attention"),
])
def test_strict_loading_names_the_key(ckpt, tmp_path, comp, gone):
    from reflectionflow_b200.transformer import B200FluxTransformer2DModel
    from reflectionflow_b200.vae import B200AutoencoderKL
    src = os.path.join(ckpt["one"], comp)
    extra = "transformer_blocks.0.attn.to_x.weight" if comp == "transformer" else "decoder.extra_block.weight"
    load = (lambda d: B200FluxTransformer2DModel.from_pretrained(d)) if comp == "transformer" else \
        (lambda d: B200AutoencoderKL.from_pretrained(d))
    missing = _rewrite(src, str(tmp_path / "missing"), lambda sd: sd.pop(gone))
    with pytest.raises(L.RFError, match=gone.replace(".", r"\.")):
        load(missing)
    added = _rewrite(src, str(tmp_path / "extra"), lambda sd: sd.update({extra: torch.zeros(4, 4)}))
    with pytest.raises(L.RFError, match=extra.replace(".", r"\.")):
        load(added)
