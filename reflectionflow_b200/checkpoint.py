"""Reading a FLUX.1-dev checkpoint in diffusers layout from disk (host side only, never the network).

What diffusers' `DiffusionPipeline.from_pretrained(name, cache_dir=...)` does before any weight reaches a
device, restated for the native components:

  * `resolve`: a local directory, or a repo id looked up in the Hugging Face hub cache by hand
    (`<cache>/models--<org>--<name>/refs/main` -> `snapshots/<revision>/`); nothing is downloaded;
  * `check_model_index`: every component the pipeline needs is named in `model_index.json` and on disk;
  * `*_config`: each component's `config.json` mapped onto what the kernels implement, refusing the rest
    before anything is allocated;
  * `SafetensorsStream`: a component's weights, one `*.safetensors` file or a sharded checkpoint with its
    `*.safetensors.index.json`, read tensor by tensor and cast to bf16 on the host, with strict key checks;
  * `tokenizer_fns`: the checkpoint's own CLIP BPE / T5 sentencepiece tokenizers, called with
    FluxPipeline's arguments.
"""
from __future__ import annotations

import json
import os
from typing import Callable, Dict, Iterator, List, Optional, Tuple

import torch

PIPELINE_COMPONENTS = ("transformer", "vae", "text_encoder", "text_encoder_2", "tokenizer", "tokenizer_2",
                       "scheduler")
# file names of a component's weights, both occur in the FLUX.1-dev repo (diffusers / transformers)
WEIGHT_NAMES = ("diffusion_pytorch_model", "model")
TOKENIZER_FILES = {"tokenizer": (("vocab.json",), ("merges.txt",)),
                   "tokenizer_2": (("tokenizer.json", "spiece.model"),)}
_FLOAT_DTYPES = (torch.bfloat16, torch.float16, torch.float32)


class CheckpointError(RuntimeError):
    pass


def _missing(path: str, what: str) -> CheckpointError:
    return CheckpointError(f"{what} not found: {path} (nothing is downloaded; it must already be on disk)")


def read_json(path: str) -> dict:
    if not os.path.isfile(path):
        raise _missing(path, os.path.basename(path))
    with open(path, "r") as f:
        return json.load(f)


# ---------------------------------------------------------------------------------------------- resolution
def default_hub_cache() -> str:
    """huggingface_hub's default cache directory: $HF_HUB_CACHE, else $HF_HOME/hub, else
    ${XDG_CACHE_HOME:-~/.cache}/huggingface/hub."""
    if os.environ.get("HF_HUB_CACHE"):
        return os.environ["HF_HUB_CACHE"]
    home = os.environ.get("HF_HOME") or os.path.join(
        os.environ.get("XDG_CACHE_HOME") or os.path.join(os.path.expanduser("~"), ".cache"), "huggingface")
    return os.path.join(home, "hub")


def resolve(name_or_path: str, cache_dir: Optional[str] = None) -> str:
    """Directory holding `model_index.json`: `name_or_path` itself when it is a directory, otherwise the
    snapshot that `refs/main` names in the hub cache (`cache_dir`, or the default hub cache)."""
    name_or_path = os.fspath(name_or_path)
    if os.path.isdir(name_or_path):
        return os.path.abspath(name_or_path)
    if name_or_path.count("/") != 1 or name_or_path.startswith((".", "/")):
        raise _missing(name_or_path, "checkpoint directory")
    cache = os.fspath(cache_dir) if cache_dir is not None else default_hub_cache()
    repo = os.path.join(cache, "models--" + name_or_path.replace("/", "--"))
    ref = os.path.join(repo, "refs", "main")
    if not os.path.isfile(ref):
        raise _missing(ref, f"hub cache entry of {name_or_path}")
    with open(ref, "r") as f:
        revision = f.read().strip()
    snap = os.path.join(repo, "snapshots", revision)
    if not os.path.isdir(snap):
        raise _missing(snap, f"snapshot {revision} of {name_or_path}")
    return snap


def check_model_index(root: str) -> dict:
    """model_index.json names every component the pipeline needs, and each is a directory on disk; the
    tokenizer directories hold their vocabulary files."""
    index = read_json(os.path.join(root, "model_index.json"))
    for comp in PIPELINE_COMPONENTS:
        entry = index.get(comp)
        if not entry or entry[0] is None:
            raise CheckpointError(f"model_index.json in {root} has no `{comp}` component")
        if not os.path.isdir(os.path.join(root, comp)):
            raise _missing(os.path.join(root, comp), f"component directory `{comp}`")
    for comp, groups in TOKENIZER_FILES.items():
        for alternatives in groups:
            if not any(os.path.isfile(os.path.join(root, comp, f)) for f in alternatives):
                raise _missing(os.path.join(root, comp, alternatives[0]), f"{comp} file {' or '.join(alternatives)}")
    return index


def check_dtype(torch_dtype) -> None:
    if torch_dtype not in (torch.bfloat16, "bf16", "bfloat16"):
        raise ValueError(f"torch_dtype {torch_dtype!r} is not supported: the kernels are bf16-only "
                         "(pass torch.bfloat16 or 'bf16'; fp16 / fp32 weights on disk are cast to bf16)")


# ---------------------------------------------------------------------------------------------- configs
def _refuse(component: str, key: str, value, supported) -> None:
    raise ValueError(f"{component}/config.json: {key} = {value!r} is not implemented by the kernels "
                     f"(supported: {supported!r})")


def dit_config(cfg: dict):
    """transformer/config.json (diffusers FluxTransformer2DModel) -> FluxDiTConfig."""
    from .config import FluxDiTConfig
    checks = (("patch_size", 1), ("attention_head_dim", 128))
    for key, want in checks:
        if cfg.get(key, want) != want:
            _refuse("transformer", key, cfg[key], want)
    if list(cfg.get("axes_dims_rope", (16, 56, 56))) != [16, 56, 56]:
        _refuse("transformer", "axes_dims_rope", cfg["axes_dims_rope"], [16, 56, 56])
    if cfg.get("out_channels") not in (None, cfg.get("in_channels", 64)):
        _refuse("transformer", "out_channels", cfg["out_channels"], "in_channels")
    return FluxDiTConfig(num_layers=cfg["num_layers"], num_single_layers=cfg["num_single_layers"],
                         num_attention_heads=cfg["num_attention_heads"], attention_head_dim=128,
                         in_channels=cfg["in_channels"], joint_attention_dim=cfg["joint_attention_dim"],
                         pooled_projection_dim=cfg["pooled_projection_dim"],
                         guidance_embeds=bool(cfg.get("guidance_embeds", False)))


# the one AutoencoderKL shape rf_vae_create builds (the FLUX.1 VAE)
VAE_SHAPE = dict(latent_channels=16, block_out_channels=[128, 256, 512, 512], layers_per_block=2,
                 norm_num_groups=32, in_channels=3, out_channels=3, act_fn="silu")


def vae_config(cfg: dict) -> Dict[str, float]:
    """vae/config.json (diffusers AutoencoderKL) -> {scaling_factor, shift_factor}."""
    for key in ("use_quant_conv", "use_post_quant_conv"):
        if cfg.get(key, True):
            _refuse("vae", key, cfg.get(key, True), False)
    if not cfg.get("mid_block_add_attention", True):
        _refuse("vae", "mid_block_add_attention", False, True)
    for key, want in VAE_SHAPE.items():
        got = cfg.get(key, want)
        if (list(got) if isinstance(want, list) else got) != want:
            _refuse("vae", key, got, want)
    return {"scaling_factor": float(cfg["scaling_factor"]), "shift_factor": float(cfg.get("shift_factor") or 0.0)}


# FlowMatchEulerDiscreteScheduler options this scheduler implements, and the values the others must have
_SCHED_KEYS = ("num_train_timesteps", "shift", "use_dynamic_shifting", "base_shift", "max_shift",
               "base_image_seq_len", "max_image_seq_len")
_SCHED_DEFAULTS = {"invert_sigmas": False, "shift_terminal": None, "use_karras_sigmas": False,
                   "use_exponential_sigmas": False, "use_beta_sigmas": False, "time_shift_type": "exponential",
                   "stochastic_sampling": False}


def scheduler_config(cfg: dict) -> dict:
    """scheduler/scheduler_config.json -> the overrides FlowMatchEulerDiscreteScheduler(**overrides) takes."""
    for key, value in cfg.items():
        if key.startswith("_") or key in _SCHED_KEYS:
            continue
        if key not in _SCHED_DEFAULTS or value != _SCHED_DEFAULTS[key]:
            _refuse("scheduler", key, value, _SCHED_DEFAULTS.get(key, "absent"))
    return {k: cfg[k] for k in _SCHED_KEYS if k in cfg}


def text_config(clip: dict, t5: dict) -> Tuple[dict, int]:
    """text_encoder/config.json (CLIPTextConfig) and text_encoder_2/config.json (T5Config) -> (the
    B200TextEncoders / _TextCfg fields, CLIP's eos_token_id)."""
    if clip.get("hidden_act", "quick_gelu") != "quick_gelu":
        _refuse("text_encoder", "hidden_act", clip["hidden_act"], "quick_gelu")
    if clip["intermediate_size"] != 4 * clip["hidden_size"]:
        _refuse("text_encoder", "intermediate_size", clip["intermediate_size"], 4 * clip["hidden_size"])
    if clip.get("layer_norm_eps", 1e-5) != 1e-5:
        _refuse("text_encoder", "layer_norm_eps", clip["layer_norm_eps"], 1e-5)
    if clip["hidden_size"] != 64 * clip["num_attention_heads"]:
        _refuse("text_encoder", "num_attention_heads", clip["num_attention_heads"], clip["hidden_size"] // 64)
    if t5.get("feed_forward_proj", "relu") != "gated-gelu":
        _refuse("text_encoder_2", "feed_forward_proj", t5.get("feed_forward_proj", "relu"), "gated-gelu")
    for key, want in (("d_kv", 64), ("relative_attention_num_buckets", 32), ("relative_attention_max_distance", 128)):
        if t5.get(key, want) != want:
            _refuse("text_encoder_2", key, t5[key], want)
    fields = dict(t5_layers=t5["num_layers"], t5_d_model=t5["d_model"], t5_d_ff=t5["d_ff"], t5_heads=t5["num_heads"],
                  t5_vocab=t5["vocab_size"], t5_eps=float(t5.get("layer_norm_epsilon", 1e-6)),
                  clip_layers=clip["num_hidden_layers"], clip_d_model=clip["hidden_size"],
                  clip_heads=clip["num_attention_heads"], clip_vocab=clip["vocab_size"],
                  clip_max_pos=clip["max_position_embeddings"])
    return fields, int(clip.get("eos_token_id", 2))


# ---------------------------------------------------------------------------------------------- weights
def weight_files(component_dir: str) -> Dict[str, str]:
    """{tensor key: file} of a component: a sharded checkpoint through its `*.safetensors.index.json`, else
    the single `*.safetensors` file (`diffusion_pytorch_model` or `model`)."""
    from safetensors import safe_open
    for stem in WEIGHT_NAMES:
        index = os.path.join(component_dir, stem + ".safetensors.index.json")
        if os.path.isfile(index):
            weight_map = read_json(index)["weight_map"]
            for shard in sorted(set(weight_map.values())):
                if not os.path.isfile(os.path.join(component_dir, shard)):
                    raise _missing(os.path.join(component_dir, shard), f"shard {shard} named by {index}")
            return {k: os.path.join(component_dir, v) for k, v in weight_map.items()}
    for stem in WEIGHT_NAMES:
        single = os.path.join(component_dir, stem + ".safetensors")
        if os.path.isfile(single):
            with safe_open(single, "pt") as f:
                return {k: single for k in f.keys()}
    raise _missing(os.path.join(component_dir, WEIGHT_NAMES[0] + ".safetensors"),
                   "weights (*.safetensors or *.safetensors.index.json)")


# key rules: a function key -> key to load, or None for a key on the component's allow-list (skipped);
# any other key the component cannot place is an error that names it (the C loaders name unknown keys)
def dit_key(key: str) -> Optional[str]:
    if ".lora_" in key:
        raise CheckpointError(f"unexpected key in transformer checkpoint: {key} (LoRA factors load through "
                              "load_lora_weights)")
    return key


_VAE_DEPRECATED = {".query.": ".to_q.", ".key.": ".to_k.", ".value.": ".to_v.", ".proj_attn.": ".to_out.0."}


def vae_key(key: str) -> Optional[str]:
    """diffusers AutoencoderKL keys; the deprecated attention names (query / key / value / proj_attn) are
    renamed as diffusers does on load."""
    if not key.startswith(("encoder.", "decoder.")):
        raise CheckpointError(f"unexpected key in vae checkpoint: {key}")
    if ".attentions." in key:
        for old, new in _VAE_DEPRECATED.items():
            key = key.replace(old, new)
    return key


def clip_key(key: str) -> Optional[str]:
    return None if key == "text_model.embeddings.position_ids" else key  # a buffer older transformers saved


def t5_key(key: str) -> Optional[str]:
    return None if key == "encoder.embed_tokens.weight" else key  # tied to shared.weight


class SafetensorsStream:
    """A component's checkpoint as a state dict whose `items()` reads one tensor at a time, cast to bf16 on
    the host: what the components' `load_state_dict` iterate over.

    Each tensor is read through its own `safe_open`: an open handle maps the whole shard, and every page of
    it read so far stays resident in this process until the handle closes, so one handle per shard would
    hold a whole shard (5-10 GB) in host memory by its end.  Reopening costs one header parse per tensor."""

    def __init__(self, component_dir: str, key_rule: Callable[[str], Optional[str]]):
        self.component_dir = component_dir
        self.files = weight_files(component_dir)
        self.key_rule = key_rule

    def keys(self) -> List[str]:
        return [k for k in (self.key_rule(k) for k in self.files) if k is not None]

    def items(self) -> Iterator[Tuple[str, torch.Tensor]]:
        from safetensors import safe_open
        for key, path in self.files.items():
            name = self.key_rule(key)
            if name is None:
                continue
            with safe_open(path, "pt") as f:
                if key not in f.keys():
                    raise CheckpointError(f"{os.path.basename(path)} has no tensor {key} (its index entry names it)")
                t = f.get_tensor(key)
            if t.dtype not in _FLOAT_DTYPES:
                raise CheckpointError(f"{key} in {os.path.basename(path)} is {t.dtype}; bf16, fp16 or fp32 expected")
            out = t.to(torch.bfloat16)
            del t
            yield name, out
            del out  # before the next read: this frame keeps no tensor alive across it


def max_lora_rank(path: str) -> int:
    """Largest rank of a LoRA adapter file (or of the `pytorch_lora_weights.safetensors` in a directory), read
    from the tensor headers only: no factor is loaded."""
    from safetensors import safe_open
    path = os.fspath(path)
    if os.path.isdir(path):
        path = os.path.join(path, "pytorch_lora_weights.safetensors")
    if not os.path.isfile(path):
        raise _missing(path, "LoRA adapter")
    with safe_open(path, "pt") as f:
        ranks = [f.get_slice(k).get_shape()[0] for k in f.keys() if ".lora_A" in k]
    if not ranks:
        raise CheckpointError(f"{path} holds no `.lora_A` factors")
    return int(max(ranks))


# ---------------------------------------------------------------------------------------------- tokenizers
def tokenizer_fns(root: str) -> Tuple[Callable, Callable]:
    """(tokenizer, tokenizer_2) for B200TextEncoders.as_hook, from the checkpoint's `tokenizer/` (CLIP BPE)
    and `tokenizer_2/` (T5 sentencepiece), with the arguments of diffusers FluxPipeline._get_clip_prompt_embeds
    and _get_t5_prompt_embeds.  Tokenisation stays on the host."""
    from transformers import CLIPTokenizer, T5TokenizerFast
    clip = CLIPTokenizer.from_pretrained(os.path.join(root, "tokenizer"), local_files_only=True)
    t5 = T5TokenizerFast.from_pretrained(os.path.join(root, "tokenizer_2"), local_files_only=True)

    def call(tok, prompts, max_length):
        return tok(prompts, padding="max_length", max_length=max_length, truncation=True, return_length=False,
                   return_overflowing_tokens=False, return_tensors="pt").input_ids

    return (lambda prompts, max_length: call(clip, prompts, max_length),
            lambda prompts, max_length: call(t5, prompts, max_length))
