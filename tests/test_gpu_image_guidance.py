"""-m gpu: image classifier-free guidance (`generate(..., image_guidance_scale=s)`, generate.py:250-272) on the CUDA
DiT:
  * parity with the reference golden of tests/_image_guidance_golden.py (exact mode, the project's bars);
  * rf_op_image_guidance_step equals torch's bf16 expression bit for bit;
  * s = 1 is today's loop (bytes and launches); s = 0 with U_i = C0 is the plain loop at guidance 1;
  * the captured guided loop equals an eager composition (two forwards + the op per step), exact and merged;
  * one handle switching between unguided and guided calls (and s) matches fresh handles;
  * an image Condition with a generator equals explicit latents built from the same posterior noise;
  * refusals, and the launch count of the captured guided step."""
import dataclasses
import json

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import cases as C  # noqa: E402
from oracle import flux_oracle as fo  # noqa: E402
from reflectionflow_b200 import _lib as L  # noqa: E402
from reflectionflow_b200.pipeline import B200FluxPipeline, Condition, generate  # noqa: E402
from reflectionflow_b200.transformer import B200FluxTransformer2DModel, lora_scale  # noqa: E402
from tests import _image_guidance_golden as G  # noqa: E402

SMALL = G.CASES["ig_s15"]


def _model(case, mode="exact", with_lora=True):
    model, lora = C.build_model(case)
    m = B200FluxTransformer2DModel(case.config(), lora_rank=case.lora_rank)
    m.load_state_dict(model.state_dict())
    if lora and with_lora:
        m.load_lora(lora, mode=mode)
    return m


def _denoise(m, case, s=None, U=None, guidance=None):
    """m.denoise on the case's inputs; U: [n_steps, B, n_cond, 64] (the golden layout)."""
    x = C.build_inputs(case)
    ts, sig = fo.flow_match_sigmas(case.steps, case.n_img)
    s = case.image_guidance_scale if s is None else s
    U = G.uncond_latents(case) if U is None else U
    jak = {"scale": case.lora_scale} if case.lora_scale != 1.0 else None
    with lora_scale(m, jak):
        out = m.denoise(x["latents"], x["prompt_embeds"], x["pooled"], ts.to(torch.bfloat16) / 1000, sig,
                        case.guidance if guidance is None else guidance, x["img_ids"], x["txt_ids"],
                        x["cond_latents"], x["cond_ids"], case.model_config, case.condition_scale,
                        image_guidance_scale=s, uncond_condition_latents=U.transpose(0, 1))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("name", list(G.CASES))
def test_image_guidance_matches_reference_golden(name):
    case = G.CASES[name]
    gold = G.load_golden()
    meta = json.load(open(G.GOLDEN_FILE.replace(".safetensors", ".json")))["cases"][name]
    ref, true32 = gold[name + "/bf16"].float(), gold[name + "/fp32"].float()
    m = _model(case)
    try:
        out = _denoise(m, case).float()
    finally:
        m.close()
    assert torch.isfinite(out).all()
    ours = C.golden_sample(gold, name, out)
    e_ours, e_ref, d = (ours - true32).abs(), (ref - true32).abs(), (ours - ref).abs()
    print(f"[{name}] |ours-fp32| mean {e_ours.mean():.4g} max {e_ours.max():.4g} ; |ref-fp32| mean {e_ref.mean():.4g} "
          f"max {e_ref.max():.4g} ; |ours-ref| mean {d.mean():.4g} ; guidance effect {meta['guidance_effect_mean']:.4g}"
          f" ; uncond effect {meta.get('uncond_effect_mean', 0):.4g}")
    assert e_ours.mean() <= 1.25 * e_ref.mean() + 1e-3
    assert e_ours.max() <= 2.0 * e_ref.max() + 1e-2
    assert d.mean() <= 2.0 * e_ref.mean() + 1e-3
    assert d.mean() < 0.5 * meta["guidance_effect_mean"]


@pytest.mark.parametrize("s", [0.0, 1e-3, -0.45, 1.3, 2.7, 7.5])
def test_op_matches_torch_expression(s):
    n = 4096 * 64
    g = torch.Generator().manual_seed(7)
    c, u, x = (torch.randn(n, generator=g).to(torch.bfloat16) for _ in range(3))
    sig = torch.tensor([1.0, 0.93, 0.5, 0.0], dtype=torch.float32)
    # generate.py:270 then the Euler step as rf_op_euler_step computes it
    v = u + s * (c - u)
    ref = (x.float() + (sig[2] - sig[1]) * v.float()).to(torch.bfloat16)
    dev = torch.device("cuda")
    xd, cd, ud, sd = x.to(dev), c.to(dev), u.to(dev), sig.to(dev)
    scale = torch.tensor([s], dtype=torch.float32, device=dev)
    step = torch.tensor([1], dtype=torch.int32, device=dev)
    lib = L.load()
    L.check(lib.rf_op_image_guidance_step(L.ptr(xd), L.ptr(cd), L.ptr(ud), L.ptr(scale), L.ptr(sd), L.ptr(step), n,
                                          L.cur_stream()), "rf_op_image_guidance_step")
    torch.cuda.synchronize()
    assert torch.equal(xd.cpu(), ref)


def _pipe_and_inputs(case):
    m = _model(case)
    x = C.build_inputs(case)
    kw = dict(prompt_embeds=x["prompt_embeds"], pooled_prompt_embeds=x["pooled"], latents=x["latents"],
              height=case.height, width=case.width, num_inference_steps=case.steps, guidance_scale=case.guidance,
              output_type="latent", max_sequence_length=case.n_txt)
    delta = [0, -(case.cond_size // 16)]
    return B200FluxPipeline(m), x, kw, delta


def test_scale_one_is_todays_loop():
    """s = 1 ignores uncond latents: the same bytes and the same launches as generate() without the keyword."""
    case = SMALL
    pipe, x, kw, delta = _pipe_and_inputs(case)
    lib = L.load()
    try:
        outs, counts = [], []
        for extra in ({}, {"image_guidance_scale": 1.0}):
            cond = Condition("cot", latents=x["cond_latents"], position_delta=delta,
                             uncond_latents=G.uncond_latents(case))
            generate(pipe, conditions=[cond], default_lora=True, **kw, **extra)  # capture
            torch.cuda.synchronize()
            n0 = lib.rf_launch_count()
            outs.append(generate(pipe, conditions=[cond], default_lora=True, **kw, **extra).images.cpu())
            torch.cuda.synchronize()
            counts.append(lib.rf_launch_count() - n0)
    finally:
        pipe.transformer.close()
    assert torch.equal(outs[0], outs[1])
    assert counts[0] == counts[1]


def test_scale_zero_with_c0_is_the_plain_loop_at_guidance_one():
    case = dataclasses.replace(SMALL, distinct_uncond=False)
    m = _model(case)
    try:
        guided = _denoise(m, case, s=0.0)
        plain = _denoise(m, case, s=1.0, guidance=1.0)
    finally:
        m.close()
    assert torch.equal(guided, plain)


def _eager(m, case, s):
    """Two tranformer_forward calls and rf_op_image_guidance_step per step, outside the captured loop."""
    x = C.build_inputs(case)
    ts, sig = fo.flow_match_sigmas(case.steps, case.n_img)
    U = G.uncond_latents(case).cuda()
    dev = torch.device("cuda")
    lat = x["latents"].to(dev).contiguous()
    sigd, scale = sig.to(dev), torch.tensor([s], dtype=torch.float32, device=dev)
    g = torch.full((case.batch,), case.guidance, dtype=torch.float32)
    lib = L.load()
    for i, t in enumerate(ts.to(torch.bfloat16) / 1000):
        args = (lat, x["prompt_embeds"], x["pooled"], t, x["img_ids"], x["txt_ids"])
        c = m._forward(*args, g, x["cond_latents"], x["cond_ids"], case.model_config, case.condition_scale)
        u = m._forward(*args, torch.ones_like(g), U[i], x["cond_ids"], case.model_config, case.condition_scale)
        step = torch.tensor([i], dtype=torch.int32, device=dev)
        L.check(lib.rf_op_image_guidance_step(L.ptr(lat), L.ptr(c), L.ptr(u), L.ptr(scale), L.ptr(sigd), L.ptr(step),
                                              lat.numel(), L.cur_stream()), "rf_op_image_guidance_step")
    torch.cuda.synchronize()
    return lat.cpu()


@pytest.mark.parametrize("mode", ["exact", "merged"])
def test_captured_loop_equals_eager_composition(mode):
    case = dataclasses.replace(G.CASES["ig_b2"], model_config={"latent_lora": True})
    m = _model(case, mode=mode)
    try:
        captured = _denoise(m, case)
        eager = _eager(m, case, case.image_guidance_scale)
    finally:
        m.close()
    assert torch.equal(captured, eager)


def test_one_handle_switching_guidance_matches_fresh_handles():
    case = SMALL
    seq = [1.0, 1.5, 2.0, 1.0]
    m = _model(case)
    try:
        reused = [_denoise(m, case, s=s) for s in seq]
    finally:
        m.close()
    for s, out in zip(seq, reused):
        f = _model(case)
        try:
            assert torch.equal(out, _denoise(f, case, s=s)), s
        finally:
            f.close()
    assert not torch.equal(reused[1], reused[2]) and not torch.equal(reused[0], reused[1])


def test_image_condition_with_generator_equals_explicit_latents():
    from reflectionflow_b200.vae import B200AutoencoderKL
    case = dataclasses.replace(SMALL, steps=3)
    pipe, x, kw, delta = _pipe_and_inputs(case)
    pipe.vae = B200AutoencoderKL("cuda:0").init_synthetic_weights(3)
    side = case.cond_size
    img = torch.randint(0, 256, (1, side, side, 3), generator=torch.Generator().manual_seed(4), dtype=torch.uint8)
    try:
        by_image = generate(pipe, conditions=[Condition("cot", condition=img, position_delta=delta,
                                                        generator=torch.Generator().manual_seed(11))],
                            default_lora=True, image_guidance_scale=1.5, **kw).images.cpu()
        g = torch.Generator().manual_seed(11)
        eps = [torch.randn((16, side // 8, side // 8), generator=g, dtype=torch.bfloat16)
               for _ in range(case.steps + 1)]
        toks = [pipe.encode_images(img.cuda(), eps=e)[0] for e in eps]
        explicit = Condition("cot", latents=toks[0], position_delta=delta, uncond_latents=torch.stack(toks[1:]))
        by_latents = generate(pipe, conditions=[explicit], default_lora=True, image_guidance_scale=1.5,
                              **kw).images.cpu()
        unguided = generate(pipe, conditions=[Condition("cot", latents=toks[0], position_delta=delta)],
                            default_lora=True, **kw).images.cpu()
    finally:
        pipe.transformer.close()
    assert torch.equal(by_image, by_latents)
    assert not torch.equal(by_latents, unguided)


def test_refusals():
    case = SMALL
    pipe, x, kw, delta = _pipe_and_inputs(case)
    try:
        with pytest.raises(ValueError, match="condition"):
            generate(pipe, conditions=None, image_guidance_scale=1.5, **kw)
        bad = Condition("cot", latents=x["cond_latents"], position_delta=delta,
                        uncond_latents=G.uncond_latents(case)[:-1])
        with pytest.raises(ValueError, match="uncond_latents"):
            generate(pipe, conditions=[bad], default_lora=True, image_guidance_scale=1.5, **kw)
        with pytest.raises(ValueError, match="uncond_condition_latents"):
            _denoise(pipe.transformer, case, U=G.uncond_latents(case)[:, :, :-1])
    finally:
        pipe.transformer.close()
    cfg = dataclasses.replace(case.config(), guidance_embeds=False)
    m = B200FluxTransformer2DModel(cfg).init_synthetic_weights(0)
    try:
        cond = Condition("cot", latents=x["cond_latents"], position_delta=delta)
        with pytest.raises(ValueError, match="guidance_embeds"):
            generate(B200FluxPipeline(m), conditions=[cond], image_guidance_scale=1.5, **kw)
    finally:
        m.close()


def test_guided_step_launches_two_forwards_and_one_kernel():
    """Per extra step, the plain loop runs its captured step (F + 1 launches: forward, Euler) plus one add of the
    step's modulation table; the guided loop runs its step (2 F + 1: two forwards, guidance + Euler) plus one add of
    each of its two tables."""
    lib = L.load()
    m = _model(SMALL)
    try:
        def per_step(s):
            counts = []
            for steps in (2, 4):
                case = dataclasses.replace(SMALL, steps=steps)
                _denoise(m, case, s=s)  # capture at this step count
                n0 = lib.rf_launch_count()
                _denoise(m, case, s=s)
                counts.append(lib.rf_launch_count() - n0)
            return (counts[1] - counts[0]) // 2
        plain_step = per_step(1.0) - 1
        guided_step = per_step(1.5) - 2
    finally:
        m.close()
    forward = plain_step - 1
    assert forward > 10
    assert guided_step == 2 * forward + 1, (plain_step, guided_step)
