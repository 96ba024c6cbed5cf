"""-m gpu: `latent_lora: True` (LoRA on every token that passes a target Linear, lora_controller.py:5-9) on the CUDA
DiT:
  * parity with the reference golden of tests/_latent_lora_golden.py, with the bars of test_gpu_dit.py, in exact
    and merged LoRA mode;
  * every LoRA target is applied to the right rows (one adapter per target);
  * the flag does not leak between calls on one handle, and without an adapter it changes nothing."""
import dataclasses

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import cases as C  # noqa: E402
from oracle import flux_oracle as fo  # noqa: E402
from reflectionflow_b200.transformer import B200FluxTransformer2DModel, tranformer_forward  # noqa: E402
from tests import _latent_lora_golden as G  # noqa: E402


def _model(case, lora, rank=None):
    model, _ = C.build_model(case)
    m = B200FluxTransformer2DModel(case.config(), lora_rank=case.lora_rank if rank is None else rank)
    m.load_state_dict(model.state_dict())
    if lora:
        m.load_lora(lora, mode="exact")
    return m


def _run(m, case, model_config=None):
    mc = case.model_config if model_config is None else model_config
    x = C.build_inputs(case)
    if case.steps:
        ts, sig = fo.flow_match_sigmas(case.steps, case.n_img)
        out = m.denoise(x["latents"], x["prompt_embeds"], x["pooled"], ts.to(torch.bfloat16) / 1000, sig,
                        case.guidance, x["img_ids"], x["txt_ids"], x["cond_latents"], x["cond_ids"], mc,
                        case.condition_scale)
    else:
        out = tranformer_forward(m, x["cond_latents"], x["cond_ids"], None, mc, 0, hidden_states=x["latents"],
                                 encoder_hidden_states=x["prompt_embeds"], pooled_projections=x["pooled"],
                                 timestep=x["timestep"], img_ids=x["img_ids"], txt_ids=x["txt_ids"],
                                 guidance=x["guidance"], joint_attention_kwargs=None, return_dict=False)[0]
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("name", list(G.CASES))
def test_latent_lora_matches_reference_golden(name):
    """Exact mode against the reference's bf16 output and the fp32 truth (bars of test_gpu_dit.py), then merged mode
    (fuse_lora: every LoRA'd group reads W + B A, the adaLN terms stay unfused) with the merged-mode bars."""
    case = G.CASES[name]
    gold = G.load_golden()
    ref, true32 = gold[name + "/bf16"].float(), gold[name + "/fp32"].float()
    e_ref = (ref - true32).abs()
    _, lora = C.build_model(case)
    m = _model(case, lora)
    try:
        exact = _run(m, case).float()
        m.load_lora(lora, mode="merged")
        merged = _run(m, case).float()
    finally:
        m.close()
    assert torch.isfinite(exact).all() and torch.isfinite(merged).all()
    assert not torch.equal(exact, merged), "merged mode must read the merged weights"
    for tag, full in (("exact", exact), ("merged", merged)):
        ours = C.golden_sample(gold, name, full)
        e_ours, d = (ours - true32).abs(), (ours - ref).abs()
        print(f"[{name} {tag}] |ours-fp32| mean {e_ours.mean():.4g} max {e_ours.max():.4g} ; |ref-fp32| mean "
              f"{e_ref.mean():.4g} max {e_ref.max():.4g} ; |ours-ref| mean {d.mean():.4g} ; bit-identical to "
              f"reference {(ours == ref).float().mean():.3f}")
        if tag == "exact":
            assert e_ours.mean() <= 1.25 * e_ref.mean() + 1e-3
            assert e_ours.max() <= 2.0 * e_ref.max() + 1e-2
            assert d.mean() <= 2.0 * e_ref.mean() + 1e-3
        else:
            assert e_ours.mean() <= 1.3 * e_ref.mean() + 1e-3
            assert e_ours.max() <= 2.5 * e_ref.max() + 1e-2


# (label, predicate on the module path): one adapter per LoRA target of train_flux/config.yaml:53
_TARGETS = [
    ("x_embedder", lambda k: k == "x_embedder"),
    ("double.norm1.linear", lambda k: k.startswith("transformer_blocks.") and k.endswith(".norm1.linear")),
    ("double.attn.to_q", lambda k: k.startswith("transformer_blocks.") and k.endswith(".attn.to_q")),
    ("double.attn.to_k", lambda k: k.startswith("transformer_blocks.") and k.endswith(".attn.to_k")),
    ("double.attn.to_v", lambda k: k.startswith("transformer_blocks.") and k.endswith(".attn.to_v")),
    ("double.attn.to_out.0", lambda k: k.startswith("transformer_blocks.") and k.endswith(".attn.to_out.0")),
    ("double.ff.net.2", lambda k: k.startswith("transformer_blocks.") and k.endswith(".ff.net.2")),
    ("single.norm.linear", lambda k: k.startswith("single_transformer_blocks.") and k.endswith(".norm.linear")),
    ("single.proj_mlp", lambda k: k.startswith("single_transformer_blocks.") and k.endswith(".proj_mlp")),
    ("single.proj_out", lambda k: k.startswith("single_transformer_blocks.") and k.endswith(".proj_out")),
    ("single.attn.to_q", lambda k: k.startswith("single_transformer_blocks.") and k.endswith(".attn.to_q")),
    ("single.attn.to_k", lambda k: k.startswith("single_transformer_blocks.") and k.endswith(".attn.to_k")),
    ("single.attn.to_v", lambda k: k.startswith("single_transformer_blocks.") and k.endswith(".attn.to_v")),
]


@pytest.mark.parametrize("label,pick", _TARGETS, ids=[t[0] for t in _TARGETS])
def test_each_target_is_applied_to_the_image_and_text_rows(label, pick):
    """Entry A (text-to-image with a LoRA on the image), one target at a time: the CUDA output must be much closer to
    the oracle with that adapter than to the un-adapted oracle.  An all-targets parity test could average away a
    missing single-block text range or a missing modulation term; one target cannot.  B is scaled by 4 so that even
    the q / k adapters move the output well beyond bf16 noise."""
    case = G.CASES["fwdA_ll_small"]
    model, full = C.build_model(case)
    one = {k: (a, (b.float() * 4).to(b.dtype)) for k, (a, b) in full.items() if pick(k)}
    assert len(one) == 1, label
    x = C.build_inputs(case)

    def oracle(lora):
        return fo.transformer_forward(model, x["latents"], x["prompt_embeds"], x["pooled"], x["timestep"],
                                      x["img_ids"], x["txt_ids"], x["guidance"], None, None, case.model_config,
                                      fo.LoraSet(lora, 1.0) if lora else None).float()
    ref, base = oracle(one), oracle(None)
    m = _model(case, one)
    try:
        ours = _run(m, case).float()
    finally:
        m.close()
    effect, d_with, d_without = (ref - base).abs().mean(), (ours - ref).abs().mean(), (ours - base).abs().mean()
    print(f"[{label}] adapter effect {effect:.4g} ; |ours - oracle(adapter)| {d_with:.4g} ; "
          f"|ours - oracle(none)| {d_without:.4g}")
    assert effect > 1e-2, "the adapter must matter in the oracle for this test to mean anything"
    assert d_with < 0.5 * d_without


@pytest.mark.parametrize("steps", [0, 4], ids=["forward", "denoise"])
def test_flag_does_not_leak_between_calls(steps):
    """latent_lora True -> False -> True on one handle: the False call equals a fresh handle with the flag off and
    both True calls are equal, bit for bit (eager forward and the captured denoise loop)."""
    case = dataclasses.replace(G.CASES["fwdB_ll_small"], steps=steps)
    off = {**case.model_config, "latent_lora": False}
    _, lora = C.build_model(case)
    m = _model(case, lora)
    try:
        a1, b, a2 = _run(m, case), _run(m, case, off), _run(m, case)
    finally:
        m.close()
    f = _model(case, lora)
    try:
        fresh_off = _run(f, case, off)
    finally:
        f.close()
    assert torch.equal(a1, a2)
    assert torch.equal(b, fresh_off)
    assert not torch.equal(a1, b)


@pytest.mark.parametrize("rank", [32, 0], ids=["no-adapter", "lora_rank0"])
@pytest.mark.parametrize("name", ["fwdB_ll_small", "denoiseA_ll_small"])
def test_without_adapter_the_flag_changes_nothing(name, rank):
    case = G.CASES[name]
    m = _model(case, None, rank=rank)
    try:
        on = _run(m, case)
        off = _run(m, case, {**case.model_config, "latent_lora": False})
    finally:
        m.close()
    assert torch.equal(on, off)



def test_text_to_image_with_a_lora_on_the_image_through_generate():
    """generate(pipe, conditions=None, model_config={"latent_lora": True}): plain text-to-image with the adapter on the
    image tokens, through the pipeline surface, against the reference golden of the same 4-step loop."""
    from reflectionflow_b200.pipeline import B200FluxPipeline, generate
    name = "denoiseA_ll_small"
    case = G.CASES[name]
    gold = G.load_golden()
    _, lora = C.build_model(case)
    m = _model(case, lora)
    x = C.build_inputs(case)
    try:
        pipe = B200FluxPipeline(m)
        outs = {ll: generate(pipe, conditions=None, model_config={"latent_lora": ll}, prompt_embeds=x["prompt_embeds"],
                             pooled_prompt_embeds=x["pooled"], latents=x["latents"], height=case.height,
                             width=case.width, num_inference_steps=case.steps, guidance_scale=case.guidance,
                             max_sequence_length=case.n_txt, output_type="latent").images.float().cpu()
                for ll in (True, False)}
    finally:
        m.close()
    assert not torch.equal(outs[True], outs[False])
    ref, true32 = gold[name + "/bf16"].float(), gold[name + "/fp32"].float()
    ours = C.golden_sample(gold, name, outs[True])
    e_ours, e_ref = (ours - true32).abs(), (ref - true32).abs()
    print(f"[generate {name}] |ours-fp32| mean {e_ours.mean():.4g} max {e_ours.max():.4g} ; |ref-fp32| mean "
          f"{e_ref.mean():.4g} max {e_ref.max():.4g}")
    assert e_ours.mean() <= 1.25 * e_ref.mean() + 1e-3
    assert e_ours.max() <= 2.0 * e_ref.max() + 1e-2
    assert (ours - ref).abs().mean() <= 2.0 * e_ref.mean() + 1e-3
