"""-m gpu: LoRA scaling (lora_alpha / r and joint_attention_kwargs["scale"]) and adapter ranks up to 128 on the CUDA
DiT:
  * parity with the reference golden of tests/_lora_scale_golden.py, with the bars of test_gpu_latent_lora.py, in
    exact and merged LoRA mode;
  * a zero scale gives the adapter-free output; alpha / r and the call scale are the same multiplier;
  * the call scale does not leak between calls (eager forward and the captured loop, exact and merged);
  * the second 64-deep low-rank k-block of a rank-128 adapter is read, and the padding adds nothing;
  * rank 128 runs the same launches as rank 32;
  * generate() with a scale, and load_lora_weights(<directory>)."""
import dataclasses

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import cases as C  # noqa: E402
from oracle import flux_oracle as fo  # noqa: E402
from reflectionflow_b200 import _lib  # noqa: E402
from reflectionflow_b200.transformer import B200FluxTransformer2DModel, lora_scale, tranformer_forward  # noqa: E402
from tests import _lora_scale_golden as G  # noqa: E402


def _model(case, lora, rank=None, alpha=None, mode="exact"):
    model, _ = C.build_model(case)
    m = B200FluxTransformer2DModel(case.config(), lora_rank=case.lora_rank if rank is None else rank)
    m.load_state_dict(model.state_dict())
    if lora:
        m.load_lora(lora, alpha=alpha, mode=mode)
    return m


def _run(m, case, scale=None, model_config=None):
    mc = case.model_config if model_config is None else model_config
    jak = None if scale is None else {"scale": scale}
    x = C.build_inputs(case)
    if case.steps:
        ts, sig = fo.flow_match_sigmas(case.steps, case.n_img)
        with lora_scale(m, jak):
            out = m.denoise(x["latents"], x["prompt_embeds"], x["pooled"], ts.to(torch.bfloat16) / 1000, sig,
                            case.guidance, x["img_ids"], x["txt_ids"], x["cond_latents"], x["cond_ids"], mc,
                            case.condition_scale)
    else:
        out = tranformer_forward(m, x["cond_latents"], x["cond_ids"], None, mc, 0, hidden_states=x["latents"],
                                 encoder_hidden_states=x["prompt_embeds"], pooled_projections=x["pooled"],
                                 timestep=x["timestep"], img_ids=x["img_ids"], txt_ids=x["txt_ids"],
                                 guidance=x["guidance"], joint_attention_kwargs=jak, return_dict=False)[0]
    torch.cuda.synchronize()
    return out.cpu()


def _golden_meta():
    import json
    return json.load(open(G.GOLDEN_FILE.replace(".safetensors", ".json")))["cases"]


@pytest.mark.parametrize("name", list(G.CASES))
def test_lora_scale_matches_reference_golden(name):
    """Exact mode against the reference's bf16 output and the fp32 truth, then merged mode (W + (B A) * scaling) with
    the merged-mode bars.  Where the scaling moves the reference's output well beyond its bf16 error, the output
    must also be much closer to the reference than that movement."""
    case = G.CASES[name]
    gold, meta = G.load_golden(), _golden_meta()[name]
    ref, true32 = gold[name + "/bf16"].float(), gold[name + "/fp32"].float()
    e_ref = (ref - true32).abs()
    _, lora = C.build_model(case)
    m = _model(case, lora, alpha=case.lora_alpha)
    try:
        exact = _run(m, case, case.lora_scale).float()
        m.load_lora(lora, alpha=case.lora_alpha, mode="merged")
        merged = _run(m, case, case.lora_scale).float()
    finally:
        m.close()
    assert torch.isfinite(exact).all() and torch.isfinite(merged).all()
    assert not torch.equal(exact, merged), "merged mode must read the merged weights"
    effect = meta["scale_effect_mean"]
    for tag, full in (("exact", exact), ("merged", merged)):
        ours = C.golden_sample(gold, name, full)
        e_ours, d = (ours - true32).abs(), (ours - ref).abs()
        print(f"[{name} {tag}] |ours-fp32| mean {e_ours.mean():.4g} max {e_ours.max():.4g} ; |ref-fp32| mean "
              f"{e_ref.mean():.4g} max {e_ref.max():.4g} ; |ours-ref| mean {d.mean():.4g} ; scale effect {effect:.4g}")
        if tag == "exact":
            assert e_ours.mean() <= 1.25 * e_ref.mean() + 1e-3
            assert e_ours.max() <= 2.0 * e_ref.max() + 1e-2
            assert d.mean() <= 2.0 * e_ref.mean() + 1e-3
        else:
            assert e_ours.mean() <= 1.3 * e_ref.mean() + 1e-3
            assert e_ours.max() <= 2.5 * e_ref.max() + 1e-2
        if effect > 5 * e_ref.mean():
            assert d.mean() < 0.5 * effect


@pytest.mark.parametrize("mode", ["exact", "merged"])
@pytest.mark.parametrize("steps", [0, 4], ids=["forward", "denoise"])
def test_zero_scale_equals_the_adapter_free_output(steps, mode):
    case = dataclasses.replace(G.CASES["fwdB_ll_r128"], steps=steps)
    _, lora = C.build_model(case)
    m = _model(case, lora, mode=mode)
    try:
        zero, one = _run(m, case, 0.0), _run(m, case)
    finally:
        m.close()
    f = _model(case, None)
    f.lora_mode = mode
    try:
        free = _run(f, case)
    finally:
        f.close()
    assert torch.equal(zero, free)
    assert not torch.equal(one, free)


def test_alpha_over_r_and_call_scale_are_the_same_multiplier():
    """alpha / r = 0.5 at call scale 1 equals alpha = r at call scale 0.5, bit for bit."""
    case = G.CASES["fwdB_ll_r128"]
    _, lora = C.build_model(case)
    outs = []
    for alpha, scale in ((case.lora_rank / 2, None), (None, 0.5)):
        m = _model(case, lora, alpha=alpha)
        try:
            outs.append(_run(m, case, scale))
        finally:
            m.close()
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("mode", ["exact", "merged"])
@pytest.mark.parametrize("steps", [0, 4], ids=["forward", "denoise"])
def test_scale_switching_on_one_handle_equals_fresh_handles(steps, mode):
    """0.75 -> 1 -> 0.75 on one handle: each call equals a fresh handle at that scale, bit for bit.  The captured
    step is re-captured and the merged weights re-merged when the scale changes."""
    case = dataclasses.replace(G.CASES["fwdB_ll_r128"], steps=steps)
    _, lora = C.build_model(case)
    m = _model(case, lora, mode=mode)
    try:
        a1, b, a2 = _run(m, case, 0.75), _run(m, case), _run(m, case, 0.75)
    finally:
        m.close()
    fresh = {}
    for s in (0.75, None):
        f = _model(case, lora, mode=mode)
        try:
            fresh[s] = _run(f, case, s)
        finally:
            f.close()
    assert torch.equal(a1, fresh[0.75]) and torch.equal(a2, fresh[0.75])
    assert torch.equal(b, fresh[None])
    assert not torch.equal(a1, b)


def test_the_second_low_rank_k_block_is_read():
    """A rank-128 adapter whose ranks 0-63 are zero lives only in the second 64-deep k-block: it must match the
    oracle and move the output well away from the adapter-free one.  With ranks 64-127 zero instead, it equals the
    rank-64 truncation on a lora_rank = 64 handle, bit for bit (the zero padding adds nothing)."""
    case = G.CASES["fwdB_ll_r128"]
    model, full = C.build_model(case)
    assert case.lora_rank == 128

    def zero_ranks(lo, hi):
        out = {}
        for k, (a, b) in full.items():
            a, b = a.clone(), b.clone()
            a[lo:hi] = 0
            b[:, lo:hi] = 0
            out[k] = (a, b)
        return out
    upper, lower = zero_ranks(0, 64), zero_ranks(64, 128)
    x = C.build_inputs(case)

    def oracle(lora):
        return fo.transformer_forward(model, x["latents"], x["prompt_embeds"], x["pooled"], x["timestep"],
                                      x["img_ids"], x["txt_ids"], x["guidance"], x["cond_latents"], x["cond_ids"],
                                      case.model_config, fo.LoraSet(lora, 1.0) if lora else None).float()
    ref, base = oracle(upper), oracle(None)
    m = _model(case, upper)
    try:
        ours = _run(m, case).float()
        m.load_lora(lower)
        ours_lower = _run(m, case)
    finally:
        m.close()
    effect, d_with, d_without = (ref - base).abs().mean(), (ours - ref).abs().mean(), (ours - base).abs().mean()
    print(f"[ranks 64-127] adapter effect {effect:.4g} ; |ours - oracle(adapter)| {d_with:.4g} ; "
          f"|ours - oracle(none)| {d_without:.4g}")
    assert effect > 1e-2
    assert d_with < 0.25 * d_without
    m64 = _model(case, {k: (a[:64].contiguous(), b[:, :64].contiguous()) for k, (a, b) in lower.items()}, rank=64)
    try:
        trunc = _run(m64, case)
    finally:
        m64.close()
    assert torch.equal(ours_lower, trunc)


def test_rank_128_runs_the_same_launches_as_rank_32():
    lib = _lib.load()
    case = G.CASES["fwdB_ll_r128"]
    counts = {}
    for rank in (32, 128):
        c = dataclasses.replace(case, lora_rank=rank)
        _, lora = C.build_model(c)
        m = _model(c, lora)
        try:
            _run(m, c, 0.8)  # warm-up: prepare, workspace
            n0 = lib.rf_launch_count()
            _run(m, c, 0.8)
            counts[rank] = lib.rf_launch_count() - n0
        finally:
            m.close()
    print("launches per forward:", counts)
    assert counts[32] == counts[128] > 0


def test_generate_with_a_call_scale_matches_the_reference():
    """generate(..., joint_attention_kwargs={"scale": s}) end to end against denoiseB_28_s; the scale is restored
    after the call."""
    from reflectionflow_b200.pipeline import B200FluxPipeline, generate
    from oracle.make_golden import FakeCondition
    name = "denoiseB_28_s"
    case = G.CASES[name]
    gold = G.load_golden()
    _, lora = C.build_model(case)
    m = _model(case, lora, alpha=case.lora_alpha)
    x = C.build_inputs(case)
    try:
        pipe = B200FluxPipeline(m)

        def gen(jak):
            return generate(pipe, conditions=[FakeCondition(x["cond_latents"], x["cond_ids"])], model_config={},
                            default_lora=True, joint_attention_kwargs=jak, prompt_embeds=x["prompt_embeds"],
                            pooled_prompt_embeds=x["pooled"], latents=x["latents"], height=case.height,
                            width=case.width, num_inference_steps=case.steps, guidance_scale=case.guidance,
                            max_sequence_length=case.n_txt, output_type="latent").images.float().cpu()
        scaled, plain = gen({"scale": case.lora_scale}), gen(None)
        direct = _run(m, case, case.lora_scale).float()
    finally:
        m.close()
    assert torch.equal(scaled, direct)
    assert not torch.equal(scaled, plain)
    ref, true32 = gold[name + "/bf16"].float(), gold[name + "/fp32"].float()
    ours = C.golden_sample(gold, name, scaled)
    e_ours, e_ref = (ours - true32).abs(), (ref - true32).abs()
    print(f"[generate {name}] |ours-fp32| mean {e_ours.mean():.4g} max {e_ours.max():.4g} ; |ref-fp32| mean "
          f"{e_ref.mean():.4g} max {e_ref.max():.4g}")
    assert e_ours.mean() <= 1.25 * e_ref.mean() + 1e-3
    assert e_ours.max() <= 2.0 * e_ref.max() + 1e-2
    assert (ours - ref).abs().mean() <= 2.0 * e_ref.mean() + 1e-3


def test_load_lora_weights_from_a_save_lora_directory(tmp_path):
    """train_flux's save_lora writes <dir>/pytorch_lora_weights.safetensors with peft keys; loading the directory
    gives the same output as loading the factors directly."""
    from safetensors.torch import save_file
    from reflectionflow_b200.pipeline import B200FluxPipeline
    case = G.CASES["fwdB_ll_r128"]
    _, lora = C.build_model(case)
    sd = {}
    for k, (a, b) in lora.items():
        sd[f"transformer.{k}.lora_A.weight"] = a.contiguous()
        sd[f"transformer.{k}.lora_B.weight"] = b.contiguous()
    save_file(sd, str(tmp_path / "pytorch_lora_weights.safetensors"))
    m = _model(case, None)
    try:
        B200FluxPipeline(m).load_lora_weights(str(tmp_path), alpha=case.lora_alpha)
        from_dir = _run(m, case, case.lora_scale)
    finally:
        m.close()
    d = _model(case, lora, alpha=case.lora_alpha)
    try:
        direct = _run(d, case, case.lora_scale)
    finally:
        d.close()
    assert torch.equal(from_dir, direct)
