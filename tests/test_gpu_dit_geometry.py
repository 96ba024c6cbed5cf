"""-m gpu: the CUDA DiT against the reference golden of the ragged-split masked-attention cases
(tests/_geometry_golden.py), with the ratio bars of test_gpu_dit.py::test_dit_matches_reference_golden."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import cases as C  # noqa: E402
from oracle import flux_oracle as fo  # noqa: E402
from reflectionflow_b200.transformer import B200FluxTransformer2DModel, tranformer_forward  # noqa: E402
from tests import _geometry_golden as G  # noqa: E402


def _run_cuda(case):
    model, lora = C.build_model(case)
    m = B200FluxTransformer2DModel(case.config(), lora_rank=case.lora_rank or 0)
    try:
        m.load_state_dict(model.state_dict())
        if lora:
            m.load_lora(lora)
        x = C.build_inputs(case)
        m.condition_scale = case.condition_scale
        if case.steps:
            ts, sig = fo.flow_match_sigmas(case.steps, case.n_img)
            out = m.denoise(x["latents"], x["prompt_embeds"], x["pooled"], ts.to(torch.bfloat16) / 1000, sig,
                            case.guidance, x["img_ids"], x["txt_ids"], x["cond_latents"], x["cond_ids"],
                            case.model_config, case.condition_scale)
        else:
            out = tranformer_forward(m, x["cond_latents"], x["cond_ids"], None, case.model_config, 0,
                                     hidden_states=x["latents"], encoder_hidden_states=x["prompt_embeds"],
                                     pooled_projections=x["pooled"], timestep=x["timestep"], img_ids=x["img_ids"],
                                     txt_ids=x["txt_ids"], guidance=x["guidance"], joint_attention_kwargs=None,
                                     return_dict=False)[0]
        torch.cuda.synchronize()
        return out.cpu()
    finally:
        m.close()


@pytest.mark.parametrize("name", list(G.CASES))
def test_dit_ragged_split_matches_reference_golden(name):
    gold = G.load_golden()
    ref_bf16, true32 = gold[name + "/bf16"].float(), gold[name + "/fp32"].float()
    full = _run_cuda(G.CASES[name]).float()
    assert torch.isfinite(full).all()
    ours = C.golden_sample(gold, name, full)
    assert ours.shape == ref_bf16.shape
    e_ours, e_ref, d = (ours - true32).abs(), (ref_bf16 - true32).abs(), (ours - ref_bf16).abs()
    print(f"[{name}] |ours-fp32| mean {e_ours.mean():.4g} max {e_ours.max():.4g} ; "
          f"|ref-fp32| mean {e_ref.mean():.4g} max {e_ref.max():.4g} ; |ours-ref| mean {d.mean():.4g} ; "
          f"bit-identical to reference {(ours == ref_bf16).float().mean():.3f}")
    assert e_ours.mean() <= 1.25 * e_ref.mean() + 1e-3
    assert e_ours.max() <= 2.0 * e_ref.max() + 1e-2
    assert d.mean() <= 2.0 * e_ref.mean() + 1e-3
