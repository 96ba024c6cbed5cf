"""Write a complete FLUX.1-dev-layout diffusers checkpoint with seeded random weights, for tests and for
measuring how long a full-size checkpoint takes to load.

  python tools/make_synthetic_checkpoint.py OUT [--layers 19,38] [--t5-layers 24] [--clip-layers 12]
      [--width full|reduced] [--shards 3] [--dtype bf16|fp16|fp32] [--vae-dtype fp32] [--seed 0]
      [--hub-cache DIR [--repo-id black-forest-labs/FLUX.1-dev]] [--lora DIR --lora-rank 32] [--device cuda]

OUT gets model_index.json; transformer/, vae/, text_encoder/, text_encoder_2/ with config.json and
safetensors (sharded with an index file when --shards > 1; the VAE and CLIP are always one file, as in the
FLUX.1-dev repo); scheduler/scheduler_config.json; tokenizer/ (a small CLIP BPE vocab.json / merges.txt) and
tokenizer_2/ (a T5-style Unigram tokenizer.json built with the `tokenizers` library: `</s>` appended, pad id 0).
With --hub-cache the directory is written as the snapshot of `--repo-id` in that Hugging Face hub cache
(`models--<org>--<name>/refs/main` + `snapshots/<revision>/`) and OUT is ignored.

Weights are drawn in bf16 (matrices N(0, 1/fan_in), biases 0.05 N(0, 1), norm scales 1 + 0.1 N(0, 1)) and
stored in the requested dtype, so the same --seed gives the same values in every dtype.  Every shard is
built and written before the next is drawn: host memory stays at about one shard.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from typing import Dict, List, Tuple

import torch

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}
WIDTHS = {
    "full": dict(heads=24, joint=4096, pooled=768, t5_d=4096, t5_ff=10240, t5_heads=64, t5_vocab=32128,
                 clip_d=768, clip_heads=12, clip_vocab=49408),
    "reduced": dict(heads=2, joint=256, pooled=256, t5_d=256, t5_ff=512, t5_heads=4, t5_vocab=1024,
                    clip_d=256, clip_heads=4, clip_vocab=1024),
}
REVISION = "0123456789abcdef0123456789abcdef01234567"
WORDS = ("a photo of the an and with on in under next to red green blue yellow white black cube sphere "
         "cat dog car tree house person two three small large image painting bright dark").split()

# public values of the FLUX.1-dev repo's config files
SCHEDULER = {"_class_name": "FlowMatchEulerDiscreteScheduler", "_diffusers_version": "0.30.0.dev0",
             "base_image_seq_len": 256, "base_shift": 0.5, "max_image_seq_len": 4096, "max_shift": 1.15,
             "num_train_timesteps": 1000, "shift": 3.0, "use_dynamic_shifting": True}
MODEL_INDEX = {"_class_name": "FluxPipeline", "_diffusers_version": "0.30.0.dev0",
               "scheduler": ["diffusers", "FlowMatchEulerDiscreteScheduler"],
               "text_encoder": ["transformers", "CLIPTextModel"], "text_encoder_2": ["transformers", "T5EncoderModel"],
               "tokenizer": ["transformers", "CLIPTokenizer"], "tokenizer_2": ["transformers", "T5TokenizerFast"],
               "transformer": ["diffusers", "FluxTransformer2DModel"], "vae": ["diffusers", "AutoencoderKL"]}
VAE_CONFIG = {"_class_name": "AutoencoderKL", "_diffusers_version": "0.30.0.dev0", "act_fn": "silu",
              "block_out_channels": [128, 256, 512, 512], "down_block_types": ["DownEncoderBlock2D"] * 4,
              "force_upcast": True, "in_channels": 3, "latent_channels": 16, "latents_mean": None, "latents_std": None,
              "layers_per_block": 2, "mid_block_add_attention": True, "norm_num_groups": 32, "out_channels": 3,
              "sample_size": 1024, "scaling_factor": 0.3611, "shift_factor": 0.1159,
              "up_block_types": ["UpDecoderBlock2D"] * 4, "use_post_quant_conv": False, "use_quant_conv": False}


# ---------------------------------------------------------------------------------------------- configs
def configs(layers=(19, 38), t5_layers=24, clip_layers=12, width="full") -> Dict[str, dict]:
    w = WIDTHS[width]
    return {
        "transformer": {"_class_name": "FluxTransformer2DModel", "_diffusers_version": "0.30.0.dev0",
                        "attention_head_dim": 128, "axes_dims_rope": [16, 56, 56], "guidance_embeds": True,
                        "in_channels": 64, "joint_attention_dim": w["joint"], "num_attention_heads": w["heads"],
                        "num_layers": layers[0], "num_single_layers": layers[1], "out_channels": None,
                        "patch_size": 1, "pooled_projection_dim": w["pooled"]},
        "vae": dict(VAE_CONFIG),
        "text_encoder": {"architectures": ["CLIPTextModel"], "model_type": "clip_text_model",
                         "attention_dropout": 0.0, "bos_token_id": 0, "eos_token_id": 2, "pad_token_id": 1,
                         "hidden_act": "quick_gelu", "hidden_size": w["clip_d"], "initializer_factor": 1.0,
                         "initializer_range": 0.02, "intermediate_size": 4 * w["clip_d"], "layer_norm_eps": 1e-5,
                         "max_position_embeddings": 77, "num_attention_heads": w["clip_heads"],
                         "num_hidden_layers": clip_layers, "projection_dim": w["pooled"],
                         "torch_dtype": "bfloat16", "vocab_size": w["clip_vocab"]},
        "text_encoder_2": {"architectures": ["T5EncoderModel"], "model_type": "t5", "d_ff": w["t5_ff"],
                           "d_kv": 64, "d_model": w["t5_d"], "dense_act_fn": "gelu_new", "dropout_rate": 0.1,
                           "eos_token_id": 1, "feed_forward_proj": "gated-gelu", "initializer_factor": 1.0,
                           "is_encoder_decoder": True, "is_gated_act": True, "layer_norm_epsilon": 1e-6,
                           "num_decoder_layers": t5_layers, "num_heads": w["t5_heads"], "num_layers": t5_layers,
                           "output_past": True, "pad_token_id": 0, "relative_attention_max_distance": 128,
                           "relative_attention_num_buckets": 32, "tie_word_embeddings": False,
                           "torch_dtype": "bfloat16", "use_cache": True, "vocab_size": w["t5_vocab"]},
        "scheduler": dict(SCHEDULER),
    }


# ---------------------------------------------------------------------------------------------- parameter lists
# (key, shape, kind): kind "w" matrix / conv, "b" bias, "n" norm scale, "e" embedding, "r" T5 relative bias
def dit_params(c: dict) -> List[Tuple[str, tuple, str]]:
    d, cin = c["num_attention_heads"] * 128, c["in_channels"]
    out = []

    def lin(name, o, i):
        out.extend([(name + ".weight", (o, i), "w"), (name + ".bias", (o,), "b")])

    lin("x_embedder", d, cin)
    lin("context_embedder", d, c["joint_attention_dim"])
    for e, i in (("timestep_embedder", 256), ("guidance_embedder", 256), ("text_embedder", c["pooled_projection_dim"])):
        if e != "guidance_embedder" or c["guidance_embeds"]:
            lin(f"time_text_embed.{e}.linear_1", d, i)
            lin(f"time_text_embed.{e}.linear_2", d, d)
    for b in range(c["num_layers"]):
        p = f"transformer_blocks.{b}."
        lin(p + "norm1.linear", 6 * d, d)
        lin(p + "norm1_context.linear", 6 * d, d)
        for n in ("to_q", "to_k", "to_v", "add_q_proj", "add_k_proj", "add_v_proj", "to_out.0", "to_add_out"):
            lin(p + "attn." + n, d, d)
        for n in ("norm_q", "norm_k", "norm_added_q", "norm_added_k"):
            out.append((p + "attn." + n + ".weight", (128,), "n"))
        lin(p + "ff.net.0.proj", 4 * d, d)
        lin(p + "ff.net.2", d, 4 * d)
        lin(p + "ff_context.net.0.proj", 4 * d, d)
        lin(p + "ff_context.net.2", d, 4 * d)
    for b in range(c["num_single_layers"]):
        p = f"single_transformer_blocks.{b}."
        lin(p + "norm.linear", 3 * d, d)
        for n in ("to_q", "to_k", "to_v"):
            lin(p + "attn." + n, d, d)
        out.extend([(p + "attn.norm_q.weight", (128,), "n"), (p + "attn.norm_k.weight", (128,), "n")])
        lin(p + "proj_mlp", 4 * d, d)
        lin(p + "proj_out", d, 5 * d)
    lin("norm_out.linear", 2 * d, d)
    lin("proj_out", cin, d)
    return out


def vae_params() -> List[Tuple[str, tuple, str]]:
    out = []

    def conv(k, co, ci, s):
        out.extend([(k + ".weight", (co, ci, s, s), "w"), (k + ".bias", (co,), "b")])

    def norm(k, ch):
        out.extend([(k + ".weight", (ch,), "n"), (k + ".bias", (ch,), "b")])

    def resnet(k, ci, co):
        norm(k + ".norm1", ci); conv(k + ".conv1", co, ci, 3)
        norm(k + ".norm2", co); conv(k + ".conv2", co, co, 3)
        if ci != co:
            conv(k + ".conv_shortcut", co, ci, 1)

    def mid(side):
        resnet(f"{side}.mid_block.resnets.0", 512, 512)
        a = f"{side}.mid_block.attentions.0."
        norm(a + "group_norm", 512)
        for n in ("to_q", "to_k", "to_v", "to_out.0"):
            out.extend([(a + n + ".weight", (512, 512), "w"), (a + n + ".bias", (512,), "b")])
        resnet(f"{side}.mid_block.resnets.1", 512, 512)

    conv("encoder.conv_in", 128, 3, 3)
    prev = 128
    for i, ch in enumerate((128, 256, 512, 512)):
        for j in range(2):
            resnet(f"encoder.down_blocks.{i}.resnets.{j}", prev if j == 0 else ch, ch)
        if i < 3:
            conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", ch, ch, 3)
        prev = ch
    mid("encoder")
    norm("encoder.conv_norm_out", 512)
    conv("encoder.conv_out", 32, 512, 3)
    conv("decoder.conv_in", 512, 16, 3)
    mid("decoder")
    prev = 512
    for i, ch in enumerate((512, 512, 256, 128)):
        for j in range(3):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else ch, ch)
        if i < 3:
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", ch, ch, 3)
        prev = ch
    norm("decoder.conv_norm_out", 128)
    conv("decoder.conv_out", 3, 128, 3)
    return out


def clip_params(c: dict) -> List[Tuple[str, tuple, str]]:
    C, p = c["hidden_size"], "text_model."
    out = [(p + "embeddings.token_embedding.weight", (c["vocab_size"], C), "e"),
           (p + "embeddings.position_embedding.weight", (c["max_position_embeddings"], C), "e")]
    for i in range(c["num_hidden_layers"]):
        q = f"{p}encoder.layers.{i}."
        for n, o, k in (("self_attn.q_proj", C, C), ("self_attn.k_proj", C, C), ("self_attn.v_proj", C, C),
                        ("self_attn.out_proj", C, C), ("mlp.fc1", 4 * C, C), ("mlp.fc2", C, 4 * C)):
            out.extend([(q + n + ".weight", (o, k), "w"), (q + n + ".bias", (o,), "b")])
        for n in ("layer_norm1", "layer_norm2"):
            out.extend([(q + n + ".weight", (C,), "n"), (q + n + ".bias", (C,), "b")])
    out.extend([(p + "final_layer_norm.weight", (C,), "n"), (p + "final_layer_norm.bias", (C,), "b")])
    return out


def t5_params(c: dict) -> List[Tuple[str, tuple, str]]:
    D, F, I = c["d_model"], c["d_ff"], c["num_heads"] * 64
    out = [("shared.weight", (c["vocab_size"], D), "e")]
    for i in range(c["num_layers"]):
        p = f"encoder.block.{i}.layer."
        out.extend([(p + f"0.SelfAttention.{n}.weight", (I, D), "w") for n in "qkv"])
        out.append((p + "0.SelfAttention.o.weight", (D, I), "w"))
        if i == 0:
            out.append((p + "0.SelfAttention.relative_attention_bias.weight", (32, c["num_heads"]), "r"))
        out.append((p + "0.layer_norm.weight", (D,), "n"))
        out.extend([(p + "1.DenseReluDense.wi_0.weight", (F, D), "w"), (p + "1.DenseReluDense.wi_1.weight", (F, D), "w"),
                    (p + "1.DenseReluDense.wo.weight", (D, F), "w"), (p + "1.layer_norm.weight", (D,), "n")])
    out.append(("encoder.final_layer_norm.weight", (D,), "n"))
    return out


# ---------------------------------------------------------------------------------------------- writing
def _draw(g: torch.Generator, shape: tuple, kind: str, device) -> torch.Tensor:
    x = torch.randn(shape, generator=g, device=device)
    if kind == "w":
        x = x * (shape[1] * (shape[2] * shape[3] if len(shape) == 4 else 1)) ** -0.5
    elif kind == "b":
        x = 0.05 * x
    elif kind == "n":
        x = 1 + 0.1 * x
    elif kind == "e":
        x = 0.5 * x
    return x.to(torch.bfloat16)


def write_weights(directory: str, stem: str, params, shards: int, dtype: torch.dtype, g: torch.Generator,
                  device="cpu", extra: Dict[str, torch.Tensor] = None) -> None:
    """`params` split into `shards` files of about equal bytes (`stem-0000i-of-0000n.safetensors` + the index
    file), or one `stem.safetensors`.  `extra` tensors are stored as given, in the last file."""
    from safetensors.torch import save_file
    nbytes = [torch.Size(s).numel() for _, s, _ in params]
    total, groups, acc = sum(nbytes), [[] for _ in range(shards)], 0
    for p, n in zip(params, nbytes):
        groups[min(shards - 1, acc * shards // total)].append(p)
        acc += n
    weight_map = {}
    for i, group in enumerate(groups):
        name = f"{stem}.safetensors" if shards == 1 else f"{stem}-{i + 1:05d}-of-{shards:05d}.safetensors"
        tensors = {k: _draw(g, s, kind, device).to(dtype).cpu() for k, s, kind in group}
        if extra and i == shards - 1:
            tensors.update(extra)
        save_file(tensors, os.path.join(directory, name), metadata={"format": "pt"})
        weight_map.update({k: name for k in tensors})
        del tensors
    if shards > 1:
        size = sum(n * torch.tensor([], dtype=dtype).element_size() for n in nbytes)
        with open(os.path.join(directory, stem + ".safetensors.index.json"), "w") as f:
            json.dump({"metadata": {"total_size": size}, "weight_map": weight_map}, f, indent=1)


def bytes_to_unicode() -> Dict[int, str]:
    """GPT-2 / CLIP byte -> printable character table."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs, n = bs[:], 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return dict(zip(bs, map(chr, cs)))


def write_clip_tokenizer(directory: str) -> None:
    """Byte-level CLIP BPE over WORDS: 512 byte tokens (with and without `</w>`), one merge chain per word,
    then <|startoftext|> and <|endoftext|> as the two largest ids (the pooling rule of eos_token_id 2 takes
    the argmax id)."""
    chars = list(bytes_to_unicode().values())
    vocab = chars + [c + "</w>" for c in chars]
    merges = []
    for w in WORDS:
        parts = list(w[:-1]) + [w[-1] + "</w>"]
        left = parts[0]
        for right in parts[1:]:
            merged = left + right
            if merged not in vocab:
                merges.append(f"{left} {right}")
                vocab.append(merged)
            left = merged
    vocab += ["<|startoftext|>", "<|endoftext|>"]
    with open(os.path.join(directory, "vocab.json"), "w") as f:
        json.dump({t: i for i, t in enumerate(vocab)}, f)
    with open(os.path.join(directory, "merges.txt"), "w") as f:
        f.write("#version: 0.2\n" + "\n".join(merges) + "\n")
    with open(os.path.join(directory, "tokenizer_config.json"), "w") as f:
        json.dump({"tokenizer_class": "CLIPTokenizer", "model_max_length": 77, "bos_token": "<|startoftext|>",
                   "eos_token": "<|endoftext|>", "pad_token": "<|endoftext|>", "unk_token": "<|endoftext|>",
                   "do_lower_case": True}, f)


def write_t5_tokenizer(directory: str) -> None:
    """T5-style Unigram tokenizer.json: <pad> 0, </s> 1, <unk> 2, then `▁word` pieces and single characters;
    Metaspace pre-tokenizer, `</s>` appended to every sequence."""
    from tokenizers import Regex, Tokenizer, decoders, models, normalizers, pre_tokenizers, processors
    pieces = [("<pad>", 0.0), ("</s>", 0.0), ("<unk>", 0.0), ("▁", -2.0)]
    pieces += [("▁" + w, -1.0 - 0.01 * i) for i, w in enumerate(WORDS)]
    pieces += [(c, -5.0) for c in "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789.,!?'-"]
    tok = Tokenizer(models.Unigram(pieces, unk_id=2, byte_fallback=False))
    tok.normalizer = normalizers.Sequence([normalizers.Replace(Regex(" {2,}"), " ")])
    tok.pre_tokenizer = pre_tokenizers.Metaspace(replacement="▁", prepend_scheme="always")
    tok.decoder = decoders.Metaspace(replacement="▁", prepend_scheme="always")
    tok.post_processor = processors.TemplateProcessing(single=["$A", "</s>"], pair=["$A", "</s>", "$B", "</s>"],
                                                       special_tokens=[("</s>", 1)])
    tok.save(os.path.join(directory, "tokenizer.json"))
    with open(os.path.join(directory, "tokenizer_config.json"), "w") as f:
        json.dump({"tokenizer_class": "T5Tokenizer", "model_max_length": 512, "eos_token": "</s>",
                   "pad_token": "<pad>", "unk_token": "<unk>", "extra_ids": 0, "additional_special_tokens": []}, f)


def write_checkpoint(out: str, layers=(19, 38), t5_layers=24, clip_layers=12, width="full", shards=1,
                     dtype="bf16", vae_dtype="fp32", seed=0, hub_cache=None,
                     repo_id="black-forest-labs/FLUX.1-dev", device="cpu") -> str:
    """Write the checkpoint; returns the directory holding model_index.json."""
    if hub_cache is not None:
        repo = os.path.join(hub_cache, "models--" + repo_id.replace("/", "--"))
        os.makedirs(os.path.join(repo, "refs"), exist_ok=True)
        with open(os.path.join(repo, "refs", "main"), "w") as f:
            f.write(REVISION)
        out = os.path.join(repo, "snapshots", REVISION)
    cfgs = configs(tuple(layers), t5_layers, clip_layers, width)
    for comp in list(cfgs) + ["tokenizer", "tokenizer_2"]:
        os.makedirs(os.path.join(out, comp), exist_ok=True)
    with open(os.path.join(out, "model_index.json"), "w") as f:
        json.dump(MODEL_INDEX, f, indent=1)
    for comp, cfg in cfgs.items():
        name = "scheduler_config.json" if comp == "scheduler" else "config.json"
        with open(os.path.join(out, comp, name), "w") as f:
            json.dump(cfg, f, indent=1)
    g = torch.Generator(device=device).manual_seed(seed)
    dt = DTYPES[dtype]
    write_weights(os.path.join(out, "transformer"), "diffusion_pytorch_model", dit_params(cfgs["transformer"]),
                  shards, dt, g, device)
    write_weights(os.path.join(out, "vae"), "diffusion_pytorch_model", vae_params(), 1, DTYPES[vae_dtype], g, device)
    # the two keys on the loader's allow-list, as older transformers versions saved them
    write_weights(os.path.join(out, "text_encoder"), "model", clip_params(cfgs["text_encoder"]), 1, dt, g, device,
                  extra={"text_model.embeddings.position_ids": torch.arange(77)[None]})
    t5 = t5_params(cfgs["text_encoder_2"])
    write_weights(os.path.join(out, "text_encoder_2"), "model", t5, shards, dt, g, device)
    write_clip_tokenizer(os.path.join(out, "tokenizer"))
    write_t5_tokenizer(os.path.join(out, "tokenizer_2"))
    return out


def write_lora(directory: str, layers=(19, 38), width="full", rank=32, seed=1, targets="config") -> str:
    """`pytorch_lora_weights.safetensors` with peft keys (`transformer.<module>.lora_A.weight` / `.lora_B.weight`),
    as train_flux's save_lora writes it; factors from tts.reflectionflow.synthetic_lora."""
    from safetensors.torch import save_file
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from reflectionflow_b200.config import FluxDiTConfig
    from reflectionflow_b200.tts.reflectionflow import synthetic_lora
    w = WIDTHS[width]
    cfg = FluxDiTConfig(num_layers=layers[0], num_single_layers=layers[1], num_attention_heads=w["heads"],
                        joint_attention_dim=w["joint"], pooled_projection_dim=w["pooled"])
    sd = {}
    for mod, (a, b) in synthetic_lora(cfg, rank=rank, seed=seed, targets=targets).items():
        sd[f"transformer.{mod}.lora_A.weight"] = a.contiguous()
        sd[f"transformer.{mod}.lora_B.weight"] = b.contiguous()
    os.makedirs(directory, exist_ok=True)
    save_file(sd, os.path.join(directory, "pytorch_lora_weights.safetensors"), metadata={"format": "pt"})
    return directory


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("out", nargs="?", default=None)
    ap.add_argument("--layers", default="19,38", help="double,single DiT blocks")
    ap.add_argument("--t5-layers", type=int, default=24)
    ap.add_argument("--clip-layers", type=int, default=12)
    ap.add_argument("--width", choices=tuple(WIDTHS), default="full")
    ap.add_argument("--shards", type=int, default=1, help="files of the transformer and of T5")
    ap.add_argument("--dtype", choices=tuple(DTYPES), default="bf16")
    ap.add_argument("--vae-dtype", choices=tuple(DTYPES), default="fp32")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--hub-cache", default=None)
    ap.add_argument("--repo-id", default="black-forest-labs/FLUX.1-dev")
    ap.add_argument("--lora", default=None, help="also write a LoRA adapter directory here")
    ap.add_argument("--lora-rank", type=int, default=32)
    ap.add_argument("--device", default="cpu", help="where the random weights are drawn (cuda is faster)")
    a = ap.parse_args(argv)
    if a.out is None and a.hub_cache is None:
        ap.error("give OUT or --hub-cache")
    layers = tuple(int(v) for v in a.layers.split(","))
    root = write_checkpoint(a.out, layers, a.t5_layers, a.clip_layers, a.width, a.shards, a.dtype, a.vae_dtype,
                            a.seed, a.hub_cache, a.repo_id, a.device)
    print(root)
    if a.lora:
        print(write_lora(a.lora, layers, a.width, a.lora_rank))


if __name__ == "__main__":
    main()
