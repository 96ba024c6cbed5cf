"""-m gpu: per-step callbacks (`callback_on_step_end`, `pipe._interrupt`; generate.py:217-290) on the CUDA DiT:
  * parity with the reference golden of tests/_callback_golden.py through generate() / __call__ (the project's bars);
  * a no-op callback is bit-identical to no callback (entry A, entry B, image-guided, batch 2, merged LoRA);
  * the latents a callback sees equal an eager composition (forward + Euler op per step) after every step;
  * an interrupt stops the forwards: its latents and its launch count;
  * one capture at most per call; a handle mixing callback and plain calls matches a fresh one; the calls that close
    the step session make rf_dit_denoise_step fail with a message."""
import dataclasses
import ctypes
import json

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import cases as C  # noqa: E402
from oracle import flux_oracle as fo  # noqa: E402
from reflectionflow_b200 import _lib as L  # noqa: E402
from reflectionflow_b200.pipeline import B200FluxPipeline, Condition, generate  # noqa: E402
from reflectionflow_b200.transformer import B200FluxTransformer2DModel  # noqa: E402
from tests import _callback_golden as G  # noqa: E402

SMALL = G.CASES["cb_edit"]


def _model(case, mode="exact"):
    model, lora = C.build_model(case)
    m = B200FluxTransformer2DModel(case.config(), lora_rank=case.lora_rank)
    m.load_state_dict(model.state_dict())
    if lora:
        m.load_lora(lora, mode=mode)
    return m


def _run(pipe, case, callback="case", **extra):
    """The case through generate() (entry B; conditions=None without a condition) or, with entry="A", __call__."""
    x = C.build_inputs(case)
    kw = dict(prompt_embeds=x["prompt_embeds"], pooled_prompt_embeds=x["pooled"], latents=x["latents"],
              height=case.height, width=case.width, num_inference_steps=case.steps, guidance_scale=case.guidance,
              output_type="latent", max_sequence_length=case.n_txt,
              callback_on_step_end=G.scripted_callback(case) if callback == "case" else callback,
              callback_on_step_end_tensor_inputs=list(case.tensor_inputs))
    if extra.pop("entry", "B") == "A":
        out = pipe(**kw).images
    else:
        conds = None
        if case.cond_size:
            U = G.uncond_latents(case) if case.image_guidance_scale != 1.0 else None
            conds = [Condition("cot", latents=x["cond_latents"], position_delta=[0, -(case.cond_size // 16)],
                               uncond_latents=U)]
        jak = {"scale": case.lora_scale} if case.lora_scale != 1.0 else None
        out = generate(pipe, conditions=conds, default_lora=True, joint_attention_kwargs=jak,
                       image_guidance_scale=case.image_guidance_scale, **kw, **extra).images
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("name", list(G.CASES))
def test_callback_matches_reference_golden(name):
    case = G.CASES[name]
    gold = G.load_golden()
    meta = json.load(open(G.GOLDEN_FILE.replace(".safetensors", ".json")))["cases"][name]
    ref, true32 = gold[name + "/bf16"].float(), gold[name + "/fp32"].float()
    pipe = B200FluxPipeline(_model(case))
    try:
        out = _run(pipe, case, entry="A" if not case.cond_size else "B").float()
    finally:
        pipe.transformer.close()
    assert torch.isfinite(out).all()
    ours = C.golden_sample(gold, name, out)
    e_ours, e_ref, d = (ours - true32).abs(), (ref - true32).abs(), (ours - ref).abs()
    print(f"[{name}] |ours-fp32| mean {e_ours.mean():.4g} max {e_ours.max():.4g} ; |ref-fp32| mean {e_ref.mean():.4g} "
          f"max {e_ref.max():.4g} ; |ours-ref| mean {d.mean():.4g} ; edit effect {meta['edit_effect_mean']:.4g}")
    assert e_ours.mean() <= 1.25 * e_ref.mean() + 1e-3
    assert e_ours.max() <= 2.0 * e_ref.max() + 1e-2
    assert d.mean() <= 2.0 * e_ref.mean() + 1e-3
    if meta["edit_effect_mean"] > 0:
        assert d.mean() < 0.5 * meta["edit_effect_mean"]


def _noop(pipe, i, t, kw):
    return {}


@pytest.mark.parametrize("variant", ["entry_a", "entry_b", "image_guided", "batch2", "merged"])
def test_noop_callback_is_bit_identical_to_no_callback(variant):
    case = {"entry_a": G.CASES["cb_entry_a"], "entry_b": SMALL, "image_guided": G.CASES["cb_ig"],
            "batch2": G.CASES["cb_b2"], "merged": dataclasses.replace(SMALL, model_config={"latent_lora": True})}[variant]
    pipe = B200FluxPipeline(_model(case, mode="merged" if variant == "merged" else "exact"))
    entry = "A" if variant == "entry_a" else "B"
    try:
        with_cb = _run(pipe, case, callback=_noop, entry=entry)
        plain = _run(pipe, case, callback=None, entry=entry)
    finally:
        pipe.transformer.close()
    assert torch.equal(with_cb, plain)


def _eager(m, case, n_steps):
    """forward + rf_op_euler_step per step, outside any captured loop: the latents after each step."""
    x = C.build_inputs(case)
    ts, sig = fo.flow_match_sigmas(case.steps, case.n_img)
    dev = torch.device("cuda")
    lat = x["latents"].to(dev).contiguous()
    sigd = sig.to(dev)
    g = torch.full((case.batch,), case.guidance, dtype=torch.float32)
    lib, out = L.load(), []
    for i, t in enumerate((ts.to(torch.bfloat16) / 1000)[:n_steps]):
        v = m._forward(lat, x["prompt_embeds"], x["pooled"], t, x["img_ids"], x["txt_ids"], g, x["cond_latents"],
                       x["cond_ids"], case.model_config, case.condition_scale)
        step = torch.tensor([i], dtype=torch.int32, device=dev)
        L.check(lib.rf_op_euler_step(L.ptr(lat), L.ptr(v), L.ptr(sigd), L.ptr(step), lat.numel(), L.cur_stream()),
                "rf_op_euler_step")
        out.append(lat.cpu())
    torch.cuda.synchronize()
    return out


def test_callback_latents_equal_eager_composition_every_step():
    case = dataclasses.replace(G.CASES["cb_b2"], kind="noop")
    pipe = B200FluxPipeline(_model(case))
    seen = []

    def record(p, i, t, kw):
        seen.append((i, t.device.type, t.dtype, t.item(), kw["latents"].clone().cpu()))
        return {}
    try:
        _run(pipe, case, callback=record)
        eager = _eager(pipe.transformer, case, case.steps)
    finally:
        pipe.transformer.close()
    ts, _ = fo.flow_match_sigmas(case.steps, case.n_img)
    assert [s[:4] for s in seen] == [(i, "cuda", torch.float32, ts[i].item()) for i in range(case.steps)]
    for i, (_, _, _, _, lat) in enumerate(seen):
        assert torch.equal(lat, eager[i]), i


def test_interrupt_stops_the_forwards():
    """Interrupt after step k: the eager composition's latents after step k, and launches = begin's + (k + 1) x the
    step graph's kernels per sample."""
    case, k = G.CASES["cb_b2"], 1
    m = _model(case)
    pipe, lib = B200FluxPipeline(m), L.load()

    def stop(p, i, t, kw):
        if i == k:
            p._interrupt = True
        return {}
    try:
        _run(pipe, case, callback=_noop)  # capture
        full_step = _launches_per_step(m, case)
        n0 = lib.rf_launch_count()
        out = _run(pipe, case, callback=stop)
        n_stop = lib.rf_launch_count() - n0
        assert pipe.interrupt
        n0 = lib.rf_launch_count()
        _run(pipe, case, callback=_noop)
        n_full = lib.rf_launch_count() - n0
        eager = _eager(m, case, k + 1)
    finally:
        m.close()
    assert torch.equal(out, eager[k])
    begin = n_full - case.steps * case.batch * full_step
    assert n_stop == begin + (k + 1) * case.batch * full_step, (n_stop, n_full, full_step)


def _launches_per_step(m, case):
    """Kernels of the captured step (one sample, one step): the launch delta of one rf_dit_denoise_step at batch 1
    would need a new geometry, so it is the step graph's count divided out of two step counts of the plain loop."""
    lib = L.load()
    x = C.build_inputs(case)
    counts = []
    for steps in (2, 4):
        ts, sig = fo.flow_match_sigmas(steps, case.n_img)
        args = (x["latents"], x["prompt_embeds"], x["pooled"], ts.to(torch.bfloat16) / 1000, sig, case.guidance,
                x["img_ids"], x["txt_ids"], x["cond_latents"], x["cond_ids"], case.model_config)
        m.denoise(*args)
        torch.cuda.synchronize()
        n0 = lib.rf_launch_count()
        m.denoise(*args)
        torch.cuda.synchronize()
        counts.append(lib.rf_launch_count() - n0)
    # per extra step and sample: the captured step + one more row of each sample's step table (one add launch)
    return (counts[1] - counts[0]) // (2 * case.batch) - 1


def test_each_call_captures_at_most_once_and_handles_mix_calls():
    case = SMALL
    lib = L.load()
    pipe = B200FluxPipeline(_model(case))
    try:
        outs = []
        for cb in ("case", None, "case"):
            n0 = lib.rf_graph_capture_count()
            outs.append(_run(pipe, case, callback=cb))
            assert lib.rf_graph_capture_count() - n0 <= 1
        n0 = lib.rf_graph_capture_count()
        _run(pipe, case)
        assert lib.rf_graph_capture_count() == n0  # nothing changed: the captured step is replayed
    finally:
        pipe.transformer.close()
    for cb, out in zip(("case", None, "case"), outs):
        f = B200FluxPipeline(_model(case))
        try:
            assert torch.equal(out, _run(f, case, callback=cb)), cb
        finally:
            f.transformer.close()
    assert not torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


@pytest.mark.parametrize("closer", ["prepare", "load_lora", "lora_scale", "denoise"])
def test_closing_calls_end_the_step_session(closer):
    case = SMALL
    m = _model(case)
    x = C.build_inputs(case)
    ts, sig = fo.flow_match_sigmas(case.steps, case.n_img)
    lib, dev = L.load(), torch.device("cuda")
    try:
        m.prepare(1, x["txt_ids"], x["img_ids"], x["cond_ids"], {}, 1.0)
        tsh = (ts.to(torch.bfloat16) / 1000).contiguous().view(torch.int16)
        sig = sig.to(torch.float32).contiguous()
        pool, cond = x["pooled"].to(dev), x["cond_latents"].to(dev)
        lat, txt = x["latents"].to(dev).contiguous(), x["prompt_embeds"].to(dev).contiguous()

        def begin():
            L.check(lib.rf_dit_denoise_begin(m._h, L.ptr(pool), ctypes.c_void_p(tsh.data_ptr()),
                                             ctypes.c_void_p(sig.data_ptr()), case.steps, ctypes.c_float(3.5),
                                             L.ptr(cond), ctypes.c_float(1.0), L.cur_stream()), "begin")
            torch.cuda.synchronize()
        step = lambda i: lib.rf_dit_denoise_step(m._h, i, L.ptr(lat), L.ptr(txt), None, L.cur_stream())  # noqa
        begin()
        assert step(0) == 0
        assert step(case.steps) != 0 and "outside" in lib.rf_last_error().decode()
        assert lib.rf_dit_denoise_step(m._h, 1, None, L.ptr(txt), None, L.cur_stream()) != 0
        if closer == "prepare":
            L.check(lib.rf_dit_prepare(m._h, 1, case.n_txt, case.n_img, case.n_cond,
                                       L.ptr(x["txt_ids"].to(dev)), L.ptr(x["img_ids"].to(dev)),
                                       L.ptr(x["cond_ids"].to(dev)), 0, ctypes.c_float(1.0), L.cur_stream()), "prep")
        elif closer == "load_lora":
            m.load_lora(C.build_model(case)[1])
        elif closer == "lora_scale":
            m.set_lora_scale(0.5)
        else:
            m.denoise(x["latents"], x["prompt_embeds"], x["pooled"], ts.to(torch.bfloat16) / 1000, sig, case.guidance,
                      x["img_ids"], x["txt_ids"], x["cond_latents"], x["cond_ids"], {})
        assert step(1) != 0
        assert "no open session" in lib.rf_last_error().decode()
        torch.cuda.synchronize()
    finally:
        m.close()


def test_returned_tensor_of_another_shape_or_dtype_is_refused():
    case = SMALL
    pipe = B200FluxPipeline(_model(case))
    try:
        for bad in (lambda lat: lat[:, :-1], lambda lat: lat.float()):
            with pytest.raises(ValueError, match="latents"):
                _run(pipe, case, callback=lambda p, i, t, kw: {"latents": bad(kw["latents"])})
    finally:
        pipe.transformer.close()
