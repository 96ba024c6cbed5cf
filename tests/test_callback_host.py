"""not-gpu: the host side of per-step callbacks (`callback_on_step_end`, `pipe._interrupt`; generate.py:217-290) with
a fake step-wise transformer: argument checks, the interrupt flag, and which steps the callback sees with which t."""
import pytest
import torch

from oracle import flux_oracle as fo
from reflectionflow_b200.pipeline import B200FluxPipeline, Condition, generate
from reflectionflow_b200.transformer import run_steps
from tests.test_host_logic import FakeTransformer


class FakeStepTransformer(FakeTransformer):
    """`denoise` with the real step-wise loop (`run_steps`) over a fake step that adds 1 to the latents and records
    the T5 states it read (test-only; not a compute fallback)."""

    def denoise(self, latents, prompt_embeds, pooled, t_in, sigmas, guidance_scale, img_ids, txt_ids,
                cond_latents=None, cond_ids=None, model_config=None, condition_scale=1.0, step_hook=None):
        self.steps = []
        self.hooked = step_hook is not None

        def step(i, lat, txt):
            self.steps.append(txt)
            lat.add_(1)
        if step_hook is None:
            for i in range(t_in.numel()):
                step(i, latents, prompt_embeds)
            return latents
        return run_steps(t_in.numel(), step, step_hook, latents, prompt_embeds)


def _inputs(B=1):
    return dict(prompt_embeds=torch.randn(B, 16, 4096).to(torch.bfloat16), pooled_prompt_embeds=torch.randn(B, 768),
                latents=torch.zeros(B, 256, 64, dtype=torch.bfloat16), height=256, width=256, num_inference_steps=4,
                output_type="latent")


def test_bad_tensor_inputs_are_refused_before_any_device_work():
    ft = FakeStepTransformer()
    pipe = B200FluxPipeline(ft)
    assert B200FluxPipeline._callback_tensor_inputs == ["latents", "prompt_embeds"]
    with pytest.raises(ValueError, match="callback_on_step_end_tensor_inputs"):
        pipe(callback_on_step_end=lambda *a: {}, callback_on_step_end_tensor_inputs=["latents", "noise_pred"],
             **_inputs())
    with pytest.raises(ValueError, match="callback_on_step_end_tensor_inputs"):
        generate(pipe, conditions=None, callback_on_step_end_tensor_inputs=["pooled_prompt_embeds"], **_inputs())
    assert not hasattr(ft, "steps")


@pytest.mark.parametrize("bad", ["shape", "dtype", "not a tensor"])
@pytest.mark.parametrize("key", ["latents", "prompt_embeds"])
def test_returned_tensor_of_another_shape_or_dtype_is_refused(bad, key):
    def cb(pipe, i, t, kw):
        x = kw[key]
        return {key: {"shape": x[:, 1:], "dtype": x.float(), "not a tensor": x.tolist()}[bad]}
    pipe = B200FluxPipeline(FakeStepTransformer())
    with pytest.raises(ValueError, match=key):
        pipe(callback_on_step_end=cb, callback_on_step_end_tensor_inputs=["latents", "prompt_embeds"], **_inputs())


def test_interrupt_is_reset_at_call_start_and_stops_the_steps():
    ft = FakeStepTransformer()
    pipe = B200FluxPipeline(ft)
    pipe._interrupt = True
    out = pipe(**_inputs()).images  # no callback: the whole loop, one call
    assert not pipe.interrupt and not ft.hooked and out.float().mean() == 4
    seen = []

    def stop_after_1(p, i, t, kw):
        seen.append(i)
        p._interrupt = i == 1
        return {}
    pipe._interrupt = True
    out = generate(pipe, conditions=None, callback_on_step_end=stop_after_1, **_inputs()).images
    assert seen == [0, 1] and len(ft.steps) == 2 and pipe.interrupt
    assert out.float().mean() == 2  # the latents as they stood after step 1


@pytest.mark.parametrize("entry", ["call", "generate"])
def test_callback_sees_every_executed_step_with_the_schedule_t(entry):
    ft = FakeStepTransformer()
    pipe = B200FluxPipeline(ft)
    seen, swap = [], torch.ones(1, 16, 4096, dtype=torch.bfloat16)

    def cb(p, i, t, kw):
        assert p is pipe and set(kw) == {"latents", "prompt_embeds"}
        seen.append((i, t.dim(), t.dtype, t.item(), kw["latents"].float().mean().item()))
        out = {"latents": kw["latents"] * 2, "ignored": 0}
        if i == 1:
            out["prompt_embeds"] = swap
        return out
    kw = dict(callback_on_step_end=cb, callback_on_step_end_tensor_inputs=["latents", "prompt_embeds"], **_inputs())
    if entry == "call":
        out = pipe(**kw).images
    else:
        cond = Condition("cot", latents=torch.zeros(1, 64, 64), position_delta=[0, -8])
        out = generate(pipe, conditions=[cond], default_lora=True, **kw).images
    ts, _ = fo.flow_match_sigmas(4, 256)
    # step i adds 1, the callback doubles: 1, 3, 7, 15 seen; 30 returned
    assert seen == [(i, 0, torch.float32, ts[i].item(), 2.0 ** (i + 1) - 1) for i in range(4)]
    assert out.float().mean() == 30
    assert torch.equal(ft.steps[2], swap) and torch.equal(ft.steps[3], swap) and not torch.equal(ft.steps[1], swap)


def test_latents_returned_with_the_interrupt_are_the_result():
    """The early-stop pattern: the callback returns new latents and interrupts in the same step.  The reference pops
    the callback's latents before its interrupt check (generate.py:289, then :218), so they are the call's result."""
    ft = FakeStepTransformer()
    pipe = B200FluxPipeline(ft)

    def cb(p, i, t, kw):
        if i == 1:
            p._interrupt = True
            return {"latents": torch.full_like(kw["latents"], 7)}
        return {}
    out = generate(pipe, conditions=None, callback_on_step_end=cb, **_inputs()).images
    assert len(ft.steps) == 2 and pipe.interrupt
    assert out.float().eq(7).all()
