"""Host side of `B200FluxPipeline.from_pretrained` (reflectionflow_b200/checkpoint.py), no GPU: resolving a
diffusers-layout FLUX.1-dev directory or its hub-cache snapshot without the network, mapping each config.json
onto what the kernels implement, the checkpoint's own tokenizers called with FluxPipeline's arguments, and
streaming the weights one tensor at a time.  Fixtures are written by tools/make_synthetic_checkpoint.py."""
import importlib.util
import json
import os
import shutil
import socket

import pytest
import torch

from reflectionflow_b200 import checkpoint as ck

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_synthetic_checkpoint",
                                               os.path.join(ROOT, "tools", "make_synthetic_checkpoint.py"))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)

SMALL = dict(layers=(1, 2), t5_layers=2, clip_layers=2, width="reduced", shards=3)


@pytest.fixture(scope="module")
def ckpt(tmp_path_factory):
    base = tmp_path_factory.mktemp("ckpt")
    local = mk.write_checkpoint(str(base / "flux"), **SMALL)
    mk.write_checkpoint(None, hub_cache=str(base / "hub"), **SMALL)
    return {"local": local, "hub": str(base / "hub"), "base": base}


def _copy(ckpt, tmp_path):
    return shutil.copytree(ckpt["local"], str(tmp_path / "copy"))


def _files(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


# ---------------------------------------------------------------------------------------------- resolution
def test_local_directory_and_hub_cache_resolve_to_the_same_files(ckpt):
    local = ck.resolve(ckpt["local"])
    hub = ck.resolve("black-forest-labs/FLUX.1-dev", cache_dir=ckpt["hub"])
    assert hub.endswith(os.path.join("snapshots", mk.REVISION))
    assert _files(local) == _files(hub)
    for comp in ("transformer", "text_encoder_2", "vae"):
        a = {k: os.path.relpath(v, local) for k, v in ck.weight_files(os.path.join(local, comp)).items()}
        b = {k: os.path.relpath(v, hub) for k, v in ck.weight_files(os.path.join(hub, comp)).items()}
        assert a == b
    ck.check_model_index(hub)


def test_default_hub_cache_comes_from_the_environment(ckpt, monkeypatch):
    monkeypatch.delenv("HF_HUB_CACHE", raising=False)
    monkeypatch.setenv("HF_HOME", "/nonexistent/hf")
    assert ck.default_hub_cache() == "/nonexistent/hf/hub"
    monkeypatch.setenv("HF_HUB_CACHE", ckpt["hub"])
    assert ck.resolve("black-forest-labs/FLUX.1-dev") == ck.resolve("black-forest-labs/FLUX.1-dev", ckpt["hub"])


def test_resolution_never_touches_the_network(ckpt, monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("network access attempted")
    monkeypatch.setattr(socket, "socket", refuse)
    monkeypatch.setattr(socket, "create_connection", refuse)
    root = ck.resolve("black-forest-labs/FLUX.1-dev", cache_dir=ckpt["hub"])
    ck.check_model_index(root)
    for comp in ("transformer", "vae", "text_encoder", "text_encoder_2"):
        ck.weight_files(os.path.join(root, comp))
    tok, tok2 = ck.tokenizer_fns(root)
    assert tok(["a red cube"], 77).shape == (1, 77) and tok2(["a red cube"], 64).shape == (1, 64)


def test_missing_repo_names_what_is_missing(ckpt):
    with pytest.raises(ck.CheckpointError, match=r"models--black-forest-labs--FLUX\.1-schnell.*refs.*main"):
        ck.resolve("black-forest-labs/FLUX.1-schnell", cache_dir=ckpt["hub"])
    with pytest.raises(ck.CheckpointError, match="must already be on disk"):
        ck.resolve("/no/such/dir")


@pytest.mark.parametrize("comp", ["transformer", "text_encoder_2", "tokenizer", "scheduler"])
def test_missing_component_is_named(ckpt, tmp_path, comp):
    root = _copy(ckpt, tmp_path)
    idx = json.load(open(os.path.join(root, "model_index.json")))
    del idx[comp]
    json.dump(idx, open(os.path.join(root, "model_index.json"), "w"))
    with pytest.raises(ck.CheckpointError, match=f"`{comp}`"):
        ck.check_model_index(root)
    # listed, but the directory itself is missing
    json.dump(mk.MODEL_INDEX, open(os.path.join(root, "model_index.json"), "w"))
    shutil.rmtree(os.path.join(root, comp))
    with pytest.raises(ck.CheckpointError, match=f"`{comp}`"):
        ck.check_model_index(root)


@pytest.mark.parametrize("comp,name", [("tokenizer", "merges.txt"), ("tokenizer", "vocab.json"),
                                       ("tokenizer_2", "tokenizer.json")])
def test_missing_tokenizer_file_is_named(ckpt, tmp_path, comp, name):
    root = _copy(ckpt, tmp_path)
    os.remove(os.path.join(root, comp, name))
    with pytest.raises(ck.CheckpointError, match=name.replace(".", r"\.")):
        ck.check_model_index(root)


def test_missing_shard_and_index_entry_are_named(ckpt, tmp_path):
    root = _copy(ckpt, tmp_path)
    tdir = os.path.join(root, "transformer")
    shard = "diffusion_pytorch_model-00002-of-00003.safetensors"
    os.rename(os.path.join(tdir, shard), os.path.join(tdir, "moved"))
    with pytest.raises(ck.CheckpointError, match=shard):
        ck.weight_files(tdir)
    os.rename(os.path.join(tdir, "moved"), os.path.join(tdir, shard))
    # an index entry that names a tensor its shard does not hold
    ipath = os.path.join(tdir, "diffusion_pytorch_model.safetensors.index.json")
    index = json.load(open(ipath))
    index["weight_map"]["transformer_blocks.0.attn.to_q.weight_typo"] = shard
    json.dump(index, open(ipath, "w"))
    with pytest.raises(ck.CheckpointError, match="to_q.weight_typo"):
        list(ck.SafetensorsStream(tdir, ck.dit_key).items())
    os.remove(ipath)  # no index and no single file: the expected names are given
    for f in os.listdir(tdir):
        if f.endswith(".safetensors"):
            os.remove(os.path.join(tdir, f))
    with pytest.raises(ck.CheckpointError, match=r"diffusion_pytorch_model\.safetensors"):
        ck.weight_files(tdir)


def test_single_file_and_model_names(ckpt, tmp_path):
    """Single-file components (`diffusion_pytorch_model.safetensors`, `model.safetensors`) list every key."""
    root = ck.resolve(ckpt["local"])
    vae = ck.weight_files(os.path.join(root, "vae"))
    assert {os.path.basename(p) for p in vae.values()} == {"diffusion_pytorch_model.safetensors"}
    assert set(vae) == {k for k, _, _ in mk.vae_params()}
    clip = ck.weight_files(os.path.join(root, "text_encoder"))
    assert {os.path.basename(p) for p in clip.values()} == {"model.safetensors"}


def test_torch_dtype():
    ck.check_dtype(torch.bfloat16)
    ck.check_dtype("bf16")
    for bad in (torch.float16, torch.float32, "fp16", "fp32", None):
        with pytest.raises(ValueError, match="bf16-only"):
            ck.check_dtype(bad)


# ---------------------------------------------------------------------------------------------- configs
FLUX = mk.configs()


def test_flux_dev_configs_map_onto_the_native_shapes():
    from reflectionflow_b200.config import FluxDiTConfig
    from reflectionflow_b200.scheduler import FlowMatchEulerDiscreteScheduler
    from reflectionflow_b200.text import CLIP_L, T5_XXL
    assert ck.dit_config(FLUX["transformer"]) == FluxDiTConfig()
    assert ck.vae_config(FLUX["vae"]) == {"scaling_factor": 0.3611, "shift_factor": 0.1159}
    fields, eos = ck.text_config(FLUX["text_encoder"], FLUX["text_encoder_2"])
    assert fields == dict(T5_XXL, **CLIP_L) and eos == 2
    over = ck.scheduler_config(FLUX["scheduler"])
    assert FlowMatchEulerDiscreteScheduler(**over).config == FlowMatchEulerDiscreteScheduler().config
    # a scheduler_config.json written by a newer diffusers carries extra options at their defaults
    newer = dict(FLUX["scheduler"], invert_sigmas=False, shift_terminal=None, use_karras_sigmas=False,
                 use_exponential_sigmas=False, use_beta_sigmas=False, time_shift_type="exponential")
    assert ck.scheduler_config(newer) == over
    # values differing from FLUX.1-dev's reach the scheduler
    assert ck.scheduler_config(dict(FLUX["scheduler"], max_shift=1.2))["max_shift"] == 1.2
    assert ck.vae_config(dict(FLUX["vae"], scaling_factor=0.5, shift_factor=0.25))["scaling_factor"] == 0.5


REFUSED = [
    ("transformer", "patch_size", 2), ("transformer", "attention_head_dim", 64),
    ("transformer", "axes_dims_rope", [16, 24, 24]), ("transformer", "out_channels", 16),
    ("vae", "use_quant_conv", True), ("vae", "use_post_quant_conv", True), ("vae", "latent_channels", 4),
    ("vae", "block_out_channels", [128, 256, 512]), ("vae", "layers_per_block", 1), ("vae", "norm_num_groups", 16),
    ("text_encoder", "hidden_act", "gelu"), ("text_encoder_2", "feed_forward_proj", "relu"),
    ("text_encoder_2", "d_kv", 128), ("text_encoder_2", "relative_attention_num_buckets", 64),
    ("text_encoder_2", "relative_attention_max_distance", 256),
    ("scheduler", "use_karras_sigmas", True), ("scheduler", "stochastic_sampling", True),
]


@pytest.mark.parametrize("comp,key,value", REFUSED)
def test_unsupported_config_is_refused_by_name(comp, key, value):
    cfgs = {c: dict(v) for c, v in FLUX.items()}
    cfgs[comp][key] = value
    with pytest.raises(ValueError, match=key):
        if comp == "transformer":
            ck.dit_config(cfgs[comp])
        elif comp == "vae":
            ck.vae_config(cfgs[comp])
        elif comp == "scheduler":
            ck.scheduler_config(cfgs[comp])
        else:
            ck.text_config(cfgs["text_encoder"], cfgs["text_encoder_2"])


@pytest.mark.parametrize("comp,key,value", [REFUSED[0], REFUSED[4], REFUSED[10], REFUSED[12], REFUSED[15]])
def test_pipeline_refuses_before_allocating(ckpt, tmp_path, monkeypatch, comp, key, value):
    """from_pretrained checks every config before any component (any device memory) is created."""
    from reflectionflow_b200 import pipeline, text, transformer, vae
    root = _copy(ckpt, tmp_path)
    name = "scheduler_config.json" if comp == "scheduler" else "config.json"
    cfg = json.load(open(os.path.join(root, comp, name)))
    cfg[key] = value
    json.dump(cfg, open(os.path.join(root, comp, name), "w"))

    def no_alloc(*a, **k):
        raise AssertionError("a component was created")
    for mod, cls in ((transformer, "B200FluxTransformer2DModel"), (vae, "B200AutoencoderKL"),
                     (text, "B200TextEncoders")):
        monkeypatch.setattr(getattr(mod, cls), "__init__", no_alloc)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    with pytest.raises(ValueError, match=key):
        pipeline.B200FluxPipeline.from_pretrained(root)
    with pytest.raises(ValueError, match="bf16-only"):
        pipeline.B200FluxPipeline.from_pretrained(ckpt["local"], torch_dtype=torch.float16)


# ---------------------------------------------------------------------------------------------- tokenizers
PROMPTS = ["a photo of a red cube on a blue sphere", "two dogs next to a large yellow house"]
LONG = " ".join(["a small green tree and a bright painting of a cat"] * 60)


@pytest.mark.parametrize("prompts,max_len", [(PROMPTS[:1], 512), (PROMPTS, 512), ([LONG], 512), ([LONG, PROMPTS[0]], 256)])
def test_tokenizer_hook_ids_equal_flux_pipeline_arguments(ckpt, prompts, max_len):
    from transformers import CLIPTokenizer, T5TokenizerFast
    root = ck.resolve(ckpt["local"])
    tok, tok2 = ck.tokenizer_fns(root)
    clip = CLIPTokenizer.from_pretrained(os.path.join(root, "tokenizer"), local_files_only=True)
    t5 = T5TokenizerFast.from_pretrained(os.path.join(root, "tokenizer_2"), local_files_only=True)
    # diffusers FluxPipeline._get_clip_prompt_embeds / _get_t5_prompt_embeds
    want = clip(prompts, padding="max_length", max_length=77, truncation=True, return_overflowing_tokens=False,
                return_length=False, return_tensors="pt").input_ids
    want2 = t5(prompts, padding="max_length", max_length=max_len, truncation=True, return_length=False,
               return_overflowing_tokens=False, return_tensors="pt").input_ids
    got, got2 = tok(prompts, 77), tok2(prompts, max_len)
    assert torch.equal(got, want) and torch.equal(got2, want2)
    assert got.shape == (len(prompts), 77) and got2.shape == (len(prompts), max_len)
    vocab = json.load(open(os.path.join(root, "tokenizer", "vocab.json")))
    eos, bos = vocab["<|endoftext|>"], vocab["<|startoftext|>"]
    assert (got[:, 0] == bos).all() and (got.argmax(-1) == (got == eos).int().argmax(-1)).all()
    for row in got2:  # </s> ends the text, <pad> (id 0) after it; a long prompt is cut, keeping its </s>
        n = int((row != 0).sum())
        assert row[n - 1] == 1 and (row[n:] == 0).all()
    if prompts[0] == LONG:
        assert (got2[0] != 0).all() and got[0, -1] == eos


# ---------------------------------------------------------------------------------------------- streaming
def test_stream_holds_one_tensor_at_a_time(ckpt, monkeypatch):
    """Every tensor is read through its own safe_open handle, which is closed before the tensor is handed
    on, and no tensor read earlier is still alive when the next is read."""
    import weakref
    real = ck.__dict__.get("safe_open")
    from safetensors import safe_open as real_open
    state = {"open": 0, "max_open": 0, "live": 0, "max_live": 0, "reads": 0}

    class Counting:
        def __init__(self, *a, **k):
            self.f = real_open(*a, **k)

        def __enter__(self):
            state["open"] += 1
            state["max_open"] = max(state["max_open"], state["open"])
            self.f.__enter__()
            return self

        def __exit__(self, *e):
            state["open"] -= 1
            return self.f.__exit__(*e)

        def keys(self):
            return self.f.keys()

        def get_slice(self, k):
            return self.f.get_slice(k)

        def get_tensor(self, k):
            t = self.f.get_tensor(k)
            state["reads"] += 1
            state["live"] += 1
            state["max_live"] = max(state["max_live"], state["live"])
            weakref.finalize(t, lambda: state.__setitem__("live", state["live"] - 1))
            return t

    import safetensors
    monkeypatch.setattr(safetensors, "safe_open", Counting)
    assert real is None  # checkpoint.py imports safe_open at call time, so the patch above reaches it
    root = ck.resolve(ckpt["local"])
    for comp, rule in (("transformer", ck.dit_key), ("vae", ck.vae_key), ("text_encoder_2", ck.t5_key)):
        stream = ck.SafetensorsStream(os.path.join(root, comp), rule)
        n = 0
        for key, t in stream.items():  # a consumer that drops each tensor once it is copied
            assert t.dtype == torch.bfloat16
            n += 1
            del t
        assert n == len(stream.keys())
    assert state["max_open"] == 1 and state["max_live"] == 1 and state["reads"] > 100


def test_fp32_and_fp16_on_disk_are_cast_to_the_same_bf16(tmp_path):
    base = dict(layers=(1, 1), t5_layers=1, clip_layers=1, width="reduced", shards=2)
    dirs = {dt: mk.write_checkpoint(str(tmp_path / dt), dtype=dt, vae_dtype=dt, **base) for dt in ("bf16", "fp32")}
    for comp, rule in (("transformer", ck.dit_key), ("vae", ck.vae_key)):
        a = dict(ck.SafetensorsStream(os.path.join(dirs["bf16"], comp), rule).items())
        b = dict(ck.SafetensorsStream(os.path.join(dirs["fp32"], comp), rule).items())
        assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    assert torch.float32 in {v.dtype for v in __import__("safetensors.torch").torch.load_file(
        os.path.join(dirs["fp32"], "vae", "diffusion_pytorch_model.safetensors")).values()}


def test_key_rules():
    assert ck.vae_key("decoder.mid_block.attentions.0.query.weight") == "decoder.mid_block.attentions.0.to_q.weight"
    assert ck.vae_key("encoder.mid_block.attentions.0.proj_attn.bias") == "encoder.mid_block.attentions.0.to_out.0.bias"
    assert ck.vae_key("decoder.mid_block.attentions.0.value.weight") == "decoder.mid_block.attentions.0.to_v.weight"
    assert ck.vae_key("decoder.up_blocks.0.resnets.0.conv1.weight") == "decoder.up_blocks.0.resnets.0.conv1.weight"
    with pytest.raises(ck.CheckpointError, match="quant_conv.weight"):
        ck.vae_key("quant_conv.weight")
    with pytest.raises(ck.CheckpointError, match="to_q.lora_A.weight"):
        ck.dit_key("transformer_blocks.0.attn.to_q.lora_A.weight")
    assert ck.clip_key("text_model.embeddings.position_ids") is None
    assert ck.t5_key("encoder.embed_tokens.weight") is None
    assert ck.t5_key("shared.weight") == "shared.weight"


def test_max_lora_rank_reads_headers_only(tmp_path):
    from safetensors.torch import save_file
    save_file({"transformer.a.lora_A.weight": torch.zeros(8, 64), "transformer.a.lora_B.weight": torch.zeros(64, 8),
               "transformer.b.lora_A.weight": torch.zeros(48, 64), "transformer.b.lora_B.weight": torch.zeros(64, 48)},
              str(tmp_path / "pytorch_lora_weights.safetensors"))
    assert ck.max_lora_rank(str(tmp_path)) == 48
    assert ck.max_lora_rank(str(tmp_path / "pytorch_lora_weights.safetensors")) == 48
    with pytest.raises(ck.CheckpointError, match="LoRA adapter"):
        ck.max_lora_rank(str(tmp_path / "nope"))
