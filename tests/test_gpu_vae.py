"""-m gpu: native FLUX VAE decoder (rf_vae_decode) vs the CPU oracle (oracle/vae_oracle.py, restated
diffusers AutoencoderKL) on seeded weights and latents.  The decoder is bf16 end to end like the
reference; GroupNorm statistics, conv summation order and the materialised bf16 attention scores
differ in rounding only, so the pre-quantisation image must agree to ~1e-2 and the uint8 image to a
couple of LSBs."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import vae_oracle as vo  # noqa: E402
from oracle import flux_oracle as fo  # noqa: E402
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


@pytest.mark.parametrize("height,width", [(64, 1024), (128, 1024), (256, 256), (128, 512), (1024, 1024)])
def test_decode_matches_oracle(height, width):
    ref, ours = _models()
    g = torch.Generator().manual_seed(height * 7 + width)
    packed = torch.randn(1, (height // 16) * (width // 16), 64, generator=g).to(torch.bfloat16)
    img_pt = ours.decode_packed(packed, height, width, "pt")
    img_u8 = ours.decode_packed(packed, height, width, "u8")
    torch.cuda.synchronize()
    torch.set_num_threads(max(1, torch.get_num_threads()))
    want = vo.decode_latents(ref, packed, height, width)            # bf16 [1, 3, H, W]
    want32 = vo.decode_latents(ref.float(), packed.float(), height, width)
    ref.to(torch.bfloat16)
    d = (img_pt.cpu().float() - want.float()).abs()
    e_ref = (want.float() - want32).abs()
    e_ours = (img_pt.cpu().float() - want32).abs()
    print(f"[vae {height}x{width}] |ours-ref_bf16| mean {d.mean():.4g} max {d.max():.4g} ; "
          f"|ref-fp32| mean {e_ref.mean():.4g} ; |ours-fp32| mean {e_ours.mean():.4g} ; "
          f"absmax {want.float().abs().max():.3g}")
    assert torch.isfinite(img_pt.float()).all()
    assert e_ours.mean() <= 1.5 * e_ref.mean() + 2e-3
    assert d.mean() <= 3.0 * e_ref.mean() + 2e-3
    rim = torch.ones(height, width, dtype=torch.bool)
    rim[1:-1, 1:-1] = False  # the image's one-pixel border on its own (a bad ring column hides in the whole mean)
    print(f"  border: |ours-ref_bf16| mean {d[..., rim].mean():.4g} ; |ref-fp32| mean {e_ref[..., rim].mean():.4g} ; "
          f"|ours-fp32| mean {e_ours[..., rim].mean():.4g}")
    assert e_ours[..., rim].mean() <= 1.5 * e_ref[..., rim].mean() + 2e-3
    assert d[..., rim].mean() <= 3.0 * e_ref[..., rim].mean() + 2e-3
    u8_want = vo.postprocess_uint8(want)
    du = (img_u8.cpu().int() - u8_want.int()).abs()
    print(f"  uint8: exact {float((du == 0).float().mean()):.3f}, <=1 {float((du <= 1).float().mean()):.3f}, "
          f"max {int(du.max())}")
    assert (du <= 2).float().mean() > 0.99


@pytest.mark.parametrize("height,width,use_eps", [(256, 256, True), (128, 512, False), (512, 512, True)])
def test_encode_matches_oracle(height, width, use_eps):
    """encode_images(): preprocess -> encoder (stride-2 convs, mid attention) -> posterior sample with
    explicit eps -> shift/scale -> pack"""
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
    print(f"[vae enc {height}x{width} eps={use_eps}] |ours-ref_bf16| mean {d.mean():.4g} max {d.max():.4g} ; "
          f"|ref-fp32| mean {e_ref.mean():.4g} ; |ours-fp32| mean {e_ours.mean():.4g} ; absmax {want.float().abs().max():.3g}")
    assert got.shape == want.shape and torch.isfinite(got.float()).all()
    assert e_ours.mean() <= 1.5 * e_ref.mean() + 2e-3
    assert d.mean() <= 3.0 * e_ref.mean() + 2e-3


def test_captured_graphs_replay_the_eager_bits(monkeypatch):
    """rf_vae_decode / rf_vae_encode capture their launch sequence per geometry and replay it (csrc/vae.cu).  A replay
    must give the bits of the eager sequence whatever ran in between: decode 256x256, encode 128x512 (other geometry,
    same workspace buffers, different zero rings), decode 256x256 again (replay), then the same calls eagerly
    (RF_VAE_GRAPH=0)."""
    _, ours = _models()
    g = torch.Generator().manual_seed(5)
    lat_a = torch.randn(1, 16 * 16, 64, generator=g).to(torch.bfloat16)
    lat_b = torch.randn(1, 16 * 16, 64, generator=g).to(torch.bfloat16)
    img = torch.randint(0, 256, (1, 128, 512, 3), generator=g, dtype=torch.uint8)
    eps = torch.randn(16, 16, 64, generator=g).to(torch.bfloat16)

    def sequence():
        outs = [ours.decode_packed(lat_a, 256, 256, "u8").clone(), ours.encode_packed(img, eps=eps).clone(),
                ours.decode_packed(lat_b, 256, 256, "u8").clone(), ours.decode_packed(lat_a, 256, 256, "pt").clone(),
                ours.encode_packed(img).clone(), ours.decode_packed(lat_a, 256, 256, "u8").clone()]
        torch.cuda.synchronize()
        return outs

    monkeypatch.setenv("RF_VAE_GRAPH", "1")
    graphed = sequence()
    monkeypatch.setenv("RF_VAE_GRAPH", "0")
    eager = sequence()
    for i, (a, b) in enumerate(zip(graphed, eager)):
        assert torch.equal(a, b), f"call {i} differs between the graph replay and the eager launch sequence"
    assert torch.equal(graphed[0], graphed[5]) and not torch.equal(graphed[0], graphed[2])


@pytest.mark.parametrize("hw,out", [((1024, 1024), (512, 512)), ((256, 384), (128, 192)), ((100, 60), (37, 45))])
def test_resize_is_bit_identical_to_pil(hw, out):
    """device BICUBIC resize == PIL.Image.resize (the parent -> 512x512 condition step)"""
    import numpy as np
    from PIL import Image
    from reflectionflow_b200.resize import resize_u8
    rng = np.random.default_rng(hw[0] + out[1])
    img = rng.integers(0, 256, size=(hw[0], hw[1], 3), dtype=np.uint8)
    want = np.array(Image.fromarray(img).resize((out[1], out[0])))
    got = resize_u8(torch.from_numpy(img)[None].cuda(), out[0], out[1])[0].cpu().numpy()
    assert np.array_equal(got, want)
