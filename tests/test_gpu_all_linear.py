"""-m gpu: a LoRA on every Linear of the transformer (train/model.py:73-80 `target_modules: "all-linear"`) on the CUDA
DiT:
  * parity with the reference golden of tests/_all_linear_golden.py, in exact and merged LoRA mode;
  * each class of new target is applied to the right rows (one class at a time), ff.net.0.proj on the image rows of
    entry A without latent_lora included;
  * a zero scale gives the adapter-free output; alpha / r and the call scale are the same multiplier;
  * the captured denoise loop equals the eager per-step forward, with the embedder and modulation terms;
  * unload_lora() returns a handle to a config.yaml:53 adapter's output and launch count;
  * the launches an all-linear step adds; non-Linear modules are refused by name."""
import dataclasses

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import cases as C  # noqa: E402
from oracle import flux_oracle as fo  # noqa: E402
from reflectionflow_b200 import _lib  # noqa: E402
from reflectionflow_b200.transformer import B200FluxTransformer2DModel, lora_scale, tranformer_forward  # noqa: E402
from tests import _all_linear_golden as G  # noqa: E402


def _model(case, lora, alpha=None, mode="exact"):
    model, _ = G.build_model(case)
    m = B200FluxTransformer2DModel(case.config(), lora_rank=case.lora_rank)
    m.load_state_dict(model.state_dict())
    m.lora_mode = mode
    if lora:
        m.load_lora(lora, alpha=alpha)
    return m


def _run(m, case, scale=None, steps=None):
    """the case's forward, or its denoise loop (rf_dit_denoise: captured step) when it has steps"""
    steps = case.steps if steps is None else steps
    jak = None if scale is None or scale == 1.0 else {"scale": scale}
    x = C.build_inputs(case)
    if steps:
        ts, sig = fo.flow_match_sigmas(steps, case.n_img)
        with lora_scale(m, jak):
            out = m.denoise(x["latents"], x["prompt_embeds"], x["pooled"], ts.to(torch.bfloat16) / 1000, sig,
                            case.guidance, x["img_ids"], x["txt_ids"], x["cond_latents"], x["cond_ids"],
                            case.model_config, case.condition_scale)
    else:
        out = tranformer_forward(m, x["cond_latents"], x["cond_ids"], None, case.model_config, 0,
                                 hidden_states=x["latents"], encoder_hidden_states=x["prompt_embeds"],
                                 pooled_projections=x["pooled"], timestep=x["timestep"], img_ids=x["img_ids"],
                                 txt_ids=x["txt_ids"], guidance=x["guidance"], joint_attention_kwargs=jak,
                                 return_dict=False)[0]
    torch.cuda.synchronize()
    return out.cpu()


def _golden_meta():
    import json
    return json.load(open(G.GOLDEN_FILE.replace(".safetensors", ".json")))["cases"]


@pytest.mark.parametrize("name", list(G.CASES))
def test_all_linear_matches_reference_golden(name):
    """Exact mode against the reference's bf16 output and the fp32 truth, then merged mode with the merged-mode bars.
    The output must also be much closer to the reference than the new targets move it."""
    case = G.CASES[name]
    gold, meta = G.load_golden(), _golden_meta()[name]
    ref, true32 = gold[name + "/bf16"].float(), gold[name + "/fp32"].float()
    e_ref = (ref - true32).abs()
    _, lora = G.build_model(case)
    m = _model(case, lora, alpha=case.lora_alpha)
    try:
        exact = _run(m, case, case.lora_scale).float()
        m.load_lora(lora, alpha=case.lora_alpha, mode="merged")
        merged = _run(m, case, case.lora_scale).float()
    finally:
        m.close()
    assert torch.isfinite(exact).all() and torch.isfinite(merged).all()
    assert not torch.equal(exact, merged), "merged mode must read the merged weights"
    effect = meta["all_linear_effect_mean"]
    for tag, full in (("exact", exact), ("merged", merged)):
        ours = C.golden_sample(gold, name, full)
        e_ours, d = (ours - true32).abs(), (ours - ref).abs()
        print(f"[{name} {tag}] |ours-fp32| mean {e_ours.mean():.4g} max {e_ours.max():.4g} ; |ref-fp32| mean "
              f"{e_ref.mean():.4g} max {e_ref.max():.4g} ; |ours-ref| mean {d.mean():.4g} ; all-linear effect "
              f"{effect:.4g}")
        if tag == "exact":
            assert e_ours.mean() <= 1.25 * e_ref.mean() + 1e-3
            assert e_ours.max() <= 2.0 * e_ref.max() + 1e-2
            assert d.mean() <= 2.0 * e_ref.mean() + 1e-3
        else:
            assert e_ours.mean() <= 1.3 * e_ref.mean() + 1e-3
            assert e_ours.max() <= 2.5 * e_ref.max() + 1e-2
        assert d.mean() < 0.1 * effect


# (label, predicate on the module path, factor on B): one class of the Linears outside train_flux/config.yaml:53 at a
# time.  The text stream's output Linears reach the image only through the single block's attention: their B is
# scaled more so that they too move the output well beyond bf16 noise.
_CLASSES = [
    ("text.qkv", lambda k: ".attn.add_" in k, 4),
    ("text.to_add_out", lambda k: k.endswith(".attn.to_add_out"), 32),
    ("ff_context.in", lambda k: k.endswith(".ff_context.net.0.proj"), 32),
    ("ff_context.out", lambda k: k.endswith(".ff_context.net.2"), 32),
    ("ff.net.0.proj", lambda k: k.endswith(".ff.net.0.proj"), 4),
    ("norm1_context", lambda k: k.endswith(".norm1_context.linear"), 4),
    ("context_embedder", lambda k: k == "context_embedder", 4),
    ("timestep_embedder", lambda k: ".timestep_embedder." in k, 4),
    ("guidance_embedder", lambda k: ".guidance_embedder." in k, 4),
    ("text_embedder", lambda k: ".text_embedder." in k, 4),
    ("norm_out", lambda k: k == "norm_out.linear", 4),
    ("proj_out", lambda k: k == "proj_out", 4),
]


@pytest.mark.parametrize("label,pick,mult", _CLASSES, ids=[t[0] for t in _CLASSES])
@pytest.mark.parametrize("name", ["fwdA_al_t128", "fwdB_al_small"])
def test_each_new_target_class_is_applied(name, label, pick, mult):
    """One class of new targets at a time, entry A without latent_lora (only the always-on rows carry a LoRA; for
    ff.net.0.proj these are the image rows) and entry B: the CUDA output must be much closer to the oracle with that
    adapter than to the un-adapted oracle."""
    case = G.CASES[name]
    _, full = G.build_model(case)
    one = {k: (a, (b.float() * mult).to(b.dtype)) for k, (a, b) in full.items() if pick(k)}
    assert one, label
    ref, base = G.run_oracle(case, lora=one).float(), G.run_oracle(case, lora={}).float()
    m = _model(case, one)
    try:
        ours = _run(m, case).float()
    finally:
        m.close()
    effect, d_with, d_without = (ref - base).abs().mean(), (ours - ref).abs().mean(), (ours - base).abs().mean()
    print(f"[{name} {label}] adapter effect {effect:.4g} ; |ours - oracle(adapter)| {d_with:.4g} ; "
          f"|ours - oracle(none)| {d_without:.4g}")
    assert effect > 1e-2, "the adapter must matter in the oracle for this test to mean anything"
    assert d_with < 0.25 * d_without


def _always_only(lora, cfg):
    return G.split(cfg, lora)[1]


@pytest.mark.parametrize("mode", ["exact", "merged"])
@pytest.mark.parametrize("steps", [0, 4], ids=["forward", "denoise"])
@pytest.mark.parametrize("which", ["all-linear", "new-only"])
def test_zero_scale_equals_the_adapter_free_output(which, steps, mode):
    case = dataclasses.replace(G.CASES["fwdB_al_ll_r128"], steps=steps)
    _, lora = G.build_model(case)
    if which == "new-only":
        lora = _always_only(lora, case.config())
    m = _model(case, lora, mode=mode)
    try:
        zero, one = _run(m, case, 0.0), _run(m, case)
    finally:
        m.close()
    f = _model(case, None, mode=mode)
    try:
        free = _run(f, case)
    finally:
        f.close()
    assert torch.equal(zero, free)
    assert not torch.equal(one, free)


@pytest.mark.parametrize("which", ["all-linear", "new-only"])
def test_alpha_over_r_and_call_scale_are_the_same_multiplier(which):
    """alpha / r = 0.5 at call scale 1 equals alpha = r at call scale 0.5, bit for bit, for the new targets too."""
    case = G.CASES["fwdB_al_ll_r128"]
    _, lora = G.build_model(case)
    if which == "new-only":
        lora = _always_only(lora, case.config())
    outs = []
    for alpha, scale in ((case.lora_rank / 2, None), (None, 0.5)):
        m = _model(case, lora, alpha=alpha)
        try:
            outs.append(_run(m, case, scale))
        finally:
            m.close()
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("mode", ["exact", "merged"])
@pytest.mark.parametrize("name", ["denoiseA_al_4", "denoiseB_al_28_s"])
def test_captured_loop_equals_the_eager_steps(name, mode):
    """rf_dit_denoise (embedder and modulation terms batched over all steps before the loop, one captured step) equals
    one eager rf_dit_forward per step followed by the scheduler's Euler step, bit for bit."""
    case = G.CASES[name]
    _, lora = G.build_model(case)
    x = C.build_inputs(case)
    ts, sig = fo.flow_match_sigmas(case.steps, case.n_img)
    tb = ts.to(torch.bfloat16) / 1000
    jak = None if case.lora_scale == 1.0 else {"scale": case.lora_scale}
    m = _model(case, lora, alpha=case.lora_alpha, mode=mode)
    try:
        loop = _run(m, case, case.lora_scale)
        lat = x["latents"].cuda()
        sg = sig.cuda()
        for i in range(case.steps):
            v = tranformer_forward(m, x["cond_latents"], x["cond_ids"], None, case.model_config, 0, hidden_states=lat,
                                   encoder_hidden_states=x["prompt_embeds"], pooled_projections=x["pooled"],
                                   timestep=tb[i:i + 1], img_ids=x["img_ids"], txt_ids=x["txt_ids"],
                                   guidance=x["guidance"], joint_attention_kwargs=jak, return_dict=False)[0]
            lat = (lat.float() + (sg[i + 1] - sg[i]) * v.float()).to(torch.bfloat16)
        torch.cuda.synchronize()
        eager = lat.cpu()
    finally:
        m.close()
    assert torch.equal(loop, eager)


def _launches(m, case, steps=None):
    lib = _lib.load()
    n0 = lib.rf_launch_count()
    _run(m, case, steps=steps)
    return lib.rf_launch_count() - n0


@pytest.mark.parametrize("mode", ["exact", "merged"])
@pytest.mark.parametrize("steps", [0, 4], ids=["forward", "denoise"])
def test_unload_then_config_adapter_equals_a_fresh_handle(steps, mode):
    """all-linear adapter -> unload_lora() -> the config.yaml:53 subset: same bits and same launches as a fresh handle
    that only ever saw the subset."""
    case = dataclasses.replace(G.CASES["fwdB_al_small"], steps=steps)
    _, lora = G.build_model(case)
    sub = G.split(case.config(), lora)[0]
    m = _model(case, lora, mode=mode)
    f = _model(case, sub, mode=mode)
    try:
        everything = _run(m, case)
        m.unload_lora()
        m.load_lora(sub)
        after = _run(m, case)
        fresh = _run(f, case)
        assert _launches(m, case) == _launches(f, case)
    finally:
        m.close()
        f.close()
    assert torch.equal(after, fresh)
    assert not torch.equal(everything, fresh)


def test_unload_lora_weights_gives_the_adapter_free_output():
    from reflectionflow_b200.pipeline import B200FluxPipeline
    case = G.CASES["fwdA_al_t128"]
    _, lora = G.build_model(case)
    m = _model(case, lora)
    f = _model(case, None)
    try:
        with_lora, free = _run(m, case), _run(f, case)
        B200FluxPipeline(m).unload_lora_weights()
        assert not m.has_lora
        unloaded = _run(m, case)
    finally:
        m.close()
        f.close()
    assert torch.equal(unloaded, free)
    assert not torch.equal(with_lora, free)


@pytest.mark.parametrize("mode,added", [("exact", None), ("merged", 0)])
def test_launches_an_all_linear_step_adds(mode, added):
    """Entry B with every LoRA group fused (128 text, 256 image, 256 condition tokens).  Exact mode: the captured step
    runs the config.yaml:53 launches + one ff.net.0.proj down-projection per double block + the T and L launches of
    context_embedder and proj_out (the text groups join the existing down-projections as groups of their own).
    Merged mode: no launch added.  The per-step count is the growth of the denoise call's count from 4 to 8 steps
    (the loop's set-up adds one launch per step in both adapters)."""
    case = dataclasses.replace(G.CASES["fwdB_al_ll_r128"], model_config={}, lora_scale=1.0, lora_alpha=None)
    _, lora = G.build_model(case)
    sub = G.split(case.config(), lora)[0]
    per_step = {}
    for tag, ad in (("config", sub), ("all-linear", lora)):
        m = _model(case, ad, mode=mode)
        try:
            _run(m, case, steps=8)  # warm-up: prepare, workspace, capture
            per_step[tag] = (_launches(m, case, 8) - _launches(m, case, 4)) / 4
        finally:
            m.close()
    print(f"[{mode}] launches per step (+1 loop set-up): {per_step}")
    want = case.double + 4 if added is None else added
    assert per_step["all-linear"] - per_step["config"] == want


def test_a_non_linear_module_is_refused_by_name():
    case = G.CASES["fwdA_al_t128"]
    m = _model(case, None)
    try:
        sd = {"transformer.transformer_blocks.0.attn.norm_q.lora_A.weight": torch.zeros(8, 128, dtype=torch.bfloat16),
              "transformer.transformer_blocks.0.attn.norm_q.lora_B.weight": torch.zeros(128, 8, dtype=torch.bfloat16)}
        with pytest.raises(Exception, match="transformer_blocks.0.attn.norm_q"):
            m.load_lora(sd)
    finally:
        m.close()
