"""-m gpu: image and condition sizes that are multiples of 16 but not of the tile sizes.

The VAE convolutions cover the image with ragged 128-pixel tiles, the mid-block attention pads its keys to
whole 128-row tiles, and the condition-masked DiT attention applies its mask / bias per element in the two
tiles that straddle the main / condition split.  Each is checked here against the same references and bars
as the tile-aligned sizes (test_gpu_vae.py, test_gpu_ops.py), then end to end through the pipeline."""
import json
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import vae_oracle as vo  # noqa: E402
from reflectionflow_b200 import _lib as L  # noqa: E402
from reflectionflow_b200.vae import B200AutoencoderKL  # noqa: E402

_CACHE = {}


def _models():
    if not _CACHE:
        torch.manual_seed(0)
        ref = vo.AutoencoderKL()
        vo.init_weights_(ref, seed=0)
        ref.eval()
        ours = B200AutoencoderKL().load_state_dict(ref.state_dict())
        _CACHE["m"] = (ref, ours)
    return _CACHE["m"]


# 768x1344 / 1360x768: common FLUX sizes (latent widths 168 and 96); 1008x1008: 15876 mid-block tokens, not a
# multiple of 64 (padded keys); 208x176: small and odd in both latent sides
@pytest.mark.parametrize("height,width", [(768, 1344), (1360, 768), (1008, 1008), (208, 176)])
def test_decode_ragged_matches_oracle(height, width):
    ref, ours = _models()
    g = torch.Generator().manual_seed(height * 7 + width)
    packed = torch.randn(1, (height // 16) * (width // 16), 64, generator=g).to(torch.bfloat16)
    img_pt = ours.decode_packed(packed, height, width, "pt")
    img_u8 = ours.decode_packed(packed, height, width, "u8")
    torch.cuda.synchronize()
    assert img_pt.shape == (1, 3, height, width) and img_u8.shape == (1, height, width, 3)
    want = vo.decode_latents(ref, packed, height, width)
    want32 = vo.decode_latents(ref.float(), packed.float(), height, width)
    ref.to(torch.bfloat16)
    d = (img_pt.cpu().float() - want.float()).abs()
    e_ref = (want.float() - want32).abs()
    e_ours = (img_pt.cpu().float() - want32).abs()
    print(f"[vae {height}x{width}] |ours-ref_bf16| mean {d.mean():.4g} max {d.max():.4g} ; "
          f"|ref-fp32| mean {e_ref.mean():.4g} ; |ours-fp32| mean {e_ours.mean():.4g}")
    assert torch.isfinite(img_pt.float()).all()
    assert e_ours.mean() <= 1.5 * e_ref.mean() + 2e-3
    assert d.mean() <= 3.0 * e_ref.mean() + 2e-3
    rim = torch.ones(height, width, dtype=torch.bool)
    rim[1:-1, 1:-1] = False  # the image's one-pixel border on its own (a bad ring column hides in the whole mean)
    print(f"  border: |ours-ref_bf16| mean {d[..., rim].mean():.4g} ; |ref-fp32| mean {e_ref[..., rim].mean():.4g} ; "
          f"|ours-fp32| mean {e_ours[..., rim].mean():.4g}")
    assert e_ours[..., rim].mean() <= 1.5 * e_ref[..., rim].mean() + 2e-3
    assert d[..., rim].mean() <= 3.0 * e_ref[..., rim].mean() + 2e-3
    du = (img_u8.cpu().int() - vo.postprocess_uint8(want).int()).abs()
    print(f"  uint8: exact {float((du == 0).float().mean()):.3f}, max {int(du.max())}")
    assert (du <= 2).float().mean() > 0.99


@pytest.mark.parametrize("height,width,use_eps", [(384, 384, True), (768, 768, False), (336, 592, True),
                                                  (336, 592, False)])
def test_encode_ragged_matches_oracle(height, width, use_eps):
    """condition sizes 384 / 768 (latent sides 48 / 96) and a non-square size with odd tile counts at every level
    of the encoder, stride-2 taps included"""
    ref, ours = _models()
    g = torch.Generator().manual_seed(height + 3 * width)
    img = torch.randint(0, 256, (height, width, 3), generator=g, dtype=torch.uint8)
    eps = torch.randn(16, height // 8, width // 8, generator=g).to(torch.bfloat16) if use_eps else None
    got = ours.encode_packed(img[None], eps)
    torch.cuda.synchronize()
    want = vo.encode_images(ref, img, eps)
    want32 = vo.encode_images(ref.float(), img, eps, dtype=torch.float32)
    ref.to(torch.bfloat16)
    d = (got.cpu().float() - want.float()).abs()
    e_ref = (want.float() - want32).abs()
    e_ours = (got.cpu().float() - want32).abs()
    print(f"[vae enc {height}x{width} eps={use_eps}] |ours-ref_bf16| mean {d.mean():.4g} ; "
          f"|ref-fp32| mean {e_ref.mean():.4g} ; |ours-fp32| mean {e_ours.mean():.4g}")
    assert got.shape == want.shape and torch.isfinite(got.float()).all()
    assert e_ours.mean() <= 1.5 * e_ref.mean() + 2e-3
    assert d.mean() <= 3.0 * e_ref.mean() + 2e-3


def test_captured_graphs_replay_the_eager_bits_ragged(monkeypatch):
    """a ragged geometry's captured decode / encode replays the eager bits when interleaved with 256x256 calls that
    share the workspace buffers (different zero rings and padded key counts)"""
    _, ours = _models()
    g = torch.Generator().manual_seed(6)
    lat_a = torch.randn(1, 13 * 11, 64, generator=g).to(torch.bfloat16)   # 208x176
    lat_b = torch.randn(1, 16 * 16, 64, generator=g).to(torch.bfloat16)   # 256x256
    img = torch.randint(0, 256, (1, 336, 592, 3), generator=g, dtype=torch.uint8)
    eps = torch.randn(16, 42, 74, generator=g).to(torch.bfloat16)

    def sequence():
        outs = [ours.decode_packed(lat_a, 208, 176, "u8").clone(), ours.decode_packed(lat_b, 256, 256, "u8").clone(),
                ours.encode_packed(img, eps=eps).clone(), ours.decode_packed(lat_a, 208, 176, "pt").clone(),
                ours.decode_packed(lat_b, 256, 256, "u8").clone(), ours.decode_packed(lat_a, 208, 176, "u8").clone()]
        torch.cuda.synchronize()
        return outs

    monkeypatch.setenv("RF_VAE_GRAPH", "1")
    graphed = sequence()
    monkeypatch.setenv("RF_VAE_GRAPH", "0")
    eager = sequence()
    for i, (a, b) in enumerate(zip(graphed, eager)):
        assert torch.equal(a, b), f"call {i} differs between the graph replay and the eager launch sequence"
    assert torch.equal(graphed[0], graphed[5]) and torch.equal(graphed[1], graphed[4])


def test_decode_rejects_sizes_off_the_16_grid():
    _, ours = _models()
    with pytest.raises(L.RFError, match="multiples of 16"):
        ours.decode_packed(torch.zeros(1, 4, 64, dtype=torch.bfloat16), 40, 24, "pt")


# ------------------------------------------------------------------ condition-masked attention, ragged split
def _randn(*shape, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(*shape, generator=g).to(torch.bfloat16).to("cuda:0")


def _attn_ref(q, k, v, heads, n_main, mode, bias):
    n = q.shape[0]
    qh, kh, vh = (t.float().view(n, heads, 128).transpose(0, 1) for t in (q, k, v))
    s = qh @ kh.transpose(1, 2) / math.sqrt(128.0)
    m = torch.zeros(n, n, device=q.device)
    val = float("-inf") if mode == 2 else bias
    m[n_main:, :n_main] = val
    m[:n_main, n_main:] = val
    o = torch.softmax(s + m, dim=-1) @ vh
    return o.transpose(0, 1).reshape(n, heads * 128)


# 4544 = 512 text + 4032 image tokens (768x1344); + 576 (384x384) or 1024 (512x512) condition tokens; 220 / 64 is
# the small case (208x176 image, 77 text tokens, 128x128 condition)
@pytest.mark.parametrize("n_main,n_cond,heads", [(4544, 576, 24), (4544, 1024, 24), (220, 64, 2)])
@pytest.mark.parametrize("mode", [1, 2])
def test_attention_cond_modes_ragged_split(mode, n_main, n_cond, heads):
    lib = L.load()
    n_tok = n_main + n_cond
    inner = heads * 128
    qkv = _randn(n_tok, 3 * inner, seed=34 + n_cond)
    q, k, v = qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:]
    bias = math.log(2.0)
    out = torch.full((n_tok, inner), float("nan"), dtype=torch.bfloat16, device="cuda:0")
    rc = lib.rf_op_attention(L.ptr(q), L.ptr(k), L.ptr(v), qkv.stride(0), L.ptr(out), out.stride(0), n_tok, heads,
                             1, n_main, mode, bias, L.cur_stream())
    L.check(rc, "rf_op_attention")
    torch.cuda.synchronize()
    ref = _attn_ref(q, k, v, heads, n_main, mode, bias)
    same = (out == ref.to(torch.bfloat16)).float().mean().item()
    d = (out.float() - ref).abs()
    print(f"[attention mode {mode} split {n_main}/{n_cond}] max {d.max():.4g} mean {d.mean():.4g} "
          f"bit-identical {same:.3f}")
    assert torch.isfinite(out.float()).all()
    torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=1e-2)
    # the rows around the split (the straddling query tile) are as close as the rest
    t0 = n_main // 128 * 128
    torch.testing.assert_close(out[t0:t0 + 128].float(), ref[t0:t0 + 128], rtol=2e-2, atol=1e-2)


# ------------------------------------------------------------------ end to end
def _pipe():
    if "pipe" not in _CACHE:
        from reflectionflow_b200.config import FluxDiTConfig
        from reflectionflow_b200.pipeline import B200FluxPipeline
        _CACHE["pipe"] = B200FluxPipeline.from_synthetic(FluxDiTConfig(num_layers=1, num_single_layers=1), seed=0,
                                                         with_vae=True)
    return _CACHE["pipe"]


def _embeds(seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(1, 512, 4096, generator=g).to(torch.bfloat16).cuda(),
            torch.randn(1, 768, generator=g).to(torch.bfloat16).cuda())


def test_pipeline_call_768x1344():
    pipe = _pipe()
    pe, pooled = _embeds(1)
    img = pipe(height=768, width=1344, num_inference_steps=2, prompt_embeds=pe, pooled_prompt_embeds=pooled,
               output_type="u8", generator=torch.Generator("cpu").manual_seed(0)).images
    assert tuple(img.shape) == (1, 768, 1344, 3) and img.dtype == torch.uint8


@pytest.mark.parametrize("model_config,condition_scale", [({"union_cond_attn": False}, 1.0), ({}, 1.5)])
def test_generate_with_384_condition(model_config, condition_scale):
    """a 384x384 condition image (576 tokens) next to a 768x1344 image: n_txt + n_img = 4544, so both masked
    attention modes run with the split inside a tile"""
    from PIL import Image
    from reflectionflow_b200.pipeline import Condition, generate
    pipe = _pipe()
    pe, pooled = _embeds(2)
    g = torch.Generator().manual_seed(3)
    cond_img = Image.fromarray(torch.randint(0, 256, (384, 384, 3), generator=g, dtype=torch.uint8).numpy())
    cond = Condition("cot", condition=cond_img, eps=torch.randn(16, 48, 48, generator=g).to(torch.bfloat16))
    img = generate(pipe, conditions=[cond], model_config=model_config, condition_scale=condition_scale,
                   default_lora=True, prompt_embeds=pe, pooled_prompt_embeds=pooled, height=768, width=1344,
                   num_inference_steps=2, output_type="u8", generator=torch.Generator("cpu").manual_seed(0)).images
    assert tuple(img.shape) == (1, 768, 1344, 3)
    assert 0 < img.float().mean().item() < 255


def test_reflection_round_768x1344_condition_384(tmp_path):
    """one noise-scaling round and one reflection round of the tts loop at height 768, width 1344,
    condition_size 384: every image written has the configured size"""
    from PIL import Image
    from reflectionflow_b200.tts import noise_scaling, reflectionflow
    from reflectionflow_b200.tts.dist import DistCtx
    base = str(tmp_path)
    config = {
        "pipeline_args": {"pretrained_model_name_or_path": "black-forest-labs/FLUX.1-dev", "cache_dir": "x",
                          "torch_dtype": "bf16", "height": 768, "width": 1344, "condition_size": 384,
                          "max_sequence_length": 512, "guidance_scale": 3.5, "num_inference_steps": 2,
                          "lora_path": "LORA"},
        "verifier_args": {"name": "nvila", "model_name": "stub", "cache_dir": "x"},
        "refine_args": {"name": "openai", "choice_of_metric": "overall_score", "max_new_tokens": 64,
                        "refine_prompt_relpath": "r.txt", "reflexion_prompt_relpath": "x.txt",
                        "verifier_prompt_relpath": "v.json"},
        "search_args": {"search_method": "random", "search_branch": 1, "search_rounds": 2},
        "model": {"add_cond_attn": False, "latent_lora": False, "union_cond_attn": True},
        "reflection_args": {"run_reflection": True, "name": "openai"},
        "prompt_refiner_args": {"run_refinement": True},
        "use_low_gpu_vram": False, "batch_size_for_img_gen": 1,
    }
    cfg0 = dict(config, search_args=dict(config["search_args"], search_rounds=1))
    json.dump(cfg0, open(os.path.join(base, "cfg0.json"), "w"))
    json.dump(config, open(os.path.join(base, "cfg.json"), "w"))
    meta = os.path.join(base, "meta.jsonl")
    with open(meta, "w") as f:
        f.write(json.dumps({"prompt": "a photo of a red cube on a blue sphere", "tag": "position"}) + "\n")
    ctx = DistCtx(0, 1, "cuda:0")
    common = ["--synthetic", "--seed", "0", "--layers", "1,1"]
    noise_scaling.main(["--pipeline_config_path", os.path.join(base, "cfg0.json"), "--meta_path", meta,
                        "--output_dir", os.path.join(base, "s0")] + common, ctx=ctx)
    reflectionflow.main(["--pipeline_config_path", os.path.join(base, "cfg.json"), "--imgpath",
                         os.path.join(base, "s0"), "--output_dir", os.path.join(base, "s1")] + common, ctx=ctx)
    torch.cuda.synchronize()
    pngs = []
    for root, _, files in os.walk(os.path.join(base, "s1")):
        pngs += [os.path.join(root, f) for f in files if f.endswith(".png")]
    mid = [p for p in pngs if os.sep + "midimg" + os.sep in p]
    assert mid, "the reflection round wrote no images"
    for p in pngs:
        im = Image.open(p)
        assert im.size == (1344, 768) and im.mode == "RGB", p
