"""CPU checks of tests/_vae_ref.py, the references the VAE kernel tests (test_gpu_vae_ops.py) compare against:

  * the convolution fixtures' fp32 accumulation is exact, so bit-exactness is the right bar;
  * the references restate the oracle (oracle/vae_oracle.py, diffusers' semantics): the convolutions, GroupNorm's
    statistics, the float64 mid-block attention, and the layout steps of `decode_latents` / `encode_images` up to the
    first convolution and after the last;
  * every entry of MUTATIONS changes at least 1 % of the outputs of a fixture the GPU file runs, or every output the
    mutation can reach, so the GPU bars would notice it;
  * the ctypes declarations match the hooks' C signatures."""
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

from oracle import vae_oracle as vo
from tests import _exact as E
from tests import _vae_ref as R
from tests import test_gpu_vae_ops as G

BF = torch.bfloat16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _changed(a, b):
    return (a.to(BF).view(torch.int16) != b.to(BF).view(torch.int16)).double().mean().item()


# ------------------------------------------------------------------------------------ exactness
@pytest.mark.parametrize("cfg", sorted(G.CONV_CFG))
def test_conv_fixture_accumulation_is_exact(cfg):
    """sum |x w| <= K max|x| max|w| = taps Cin 1 / 4 < 2^15 = 2^(23 - 8) for every layer (x on k/8, w on k/32)"""
    cin, _, _, _, taps = G.CONV_CFG[cfg]
    assert taps * cin * 1.0 * 0.25 < 2.0 ** (23 - 3 - 5)
    for H, W, stride, c, res in G.CONV_CASES:
        if c == cfg and H * W <= 26 * 22:  # the small fixtures in full (conv() asserts the exactness itself)
            x, w, b, r = G._operands(H, W, stride, cfg, res, True, "cpu")
            R.conv(x, w, b, stride, None if r is None else r[..., :w.shape[0]])


# ------------------------------------------------------------------------------------ references = the oracle
@pytest.mark.parametrize("stride,k", [(1, 3), (2, 3), (1, 1)])
def test_conv_reference_is_the_oracle(stride, k):
    x, w, b, _ = G._operands(6, 10, stride, "c128" if k == 3 else "sc128_256", None, True, "cpu")
    xd = x.double().permute(2, 0, 1)[None]
    if stride == 2:
        m = vo.Downsample2D(128).double()
    else:
        m = torch.nn.Conv2d(w.shape[1], w.shape[0], k, padding=1 if k == 3 else 0).double()
    conv = m.conv if stride == 2 else m
    with torch.no_grad():
        conv.weight.copy_(w.double())
        conv.bias.copy_(b.double())
        want = m(xd)[0].permute(1, 2, 0)
    assert torch.equal(R.conv(x, w, b, stride), E.bf(want.float()))


def test_group_norm_statistics_are_torch():
    x = E.randn((6, 10, 256), 3).float() * 2 + 1
    mean, rstd = R.gn_stats(x)
    t = x.double().permute(2, 0, 1)[None]
    want = F.group_norm(t, 32, eps=1e-6)[0].permute(1, 2, 0)
    got = (x.double() - mean.repeat_interleave(8)) * rstd.repeat_interleave(8)
    assert (got - want).abs().max().item() < 1e-12


def test_mid_attention_truth_is_the_oracle():
    m = vo.VaeAttention(512)
    vo.init_weights_(m, seed=0)
    p = m.state_dict()
    x = E.randn((3, 5, 512), 4)
    with torch.no_grad():
        want = m.double()(x.double().permute(2, 0, 1)[None])[0].permute(1, 2, 0)
    assert (R.mid_attention_truth(x, p) - want).abs().max().item() < 1e-10


def _all_finite(n):
    return G._all_finite_bf16(n)


def test_unpack_reference_is_decode_latents():
    """every finite bf16 value through vo.decode_latents up to the first convolution (test_gpu_vae_ops.py runs the
    same on the GPU, where torch keeps the shift in fp32)"""
    h = w = 64
    packed = _all_finite(h * w * 16)[torch.randperm(h * w * 16, generator=torch.Generator().manual_seed(0))]
    packed = packed.view(1, (h // 2) * (w // 2), 64)
    want = vo.decode_latents(R.OracleStub(), packed, 8 * h, 8 * w)[0].permute(1, 2, 0)
    assert torch.equal(R.unpack_latents(packed[0], h, w, shift=R.SHIFT_CPU), want.float())


def test_upsample_reference_is_interpolate():
    x = E.randn((5, 7, 16), 2)
    want = F.interpolate(x.float().permute(2, 0, 1)[None], scale_factor=2.0, mode="nearest")[0].permute(1, 2, 0)
    assert torch.equal(R.upsample2x(x).float(), want)


def test_preprocess_division_is_numpy():
    """VaeImageProcessor.pil_to_numpy divides by 255 in numpy fp32 (correctly rounded), as the kernel's '/' does"""
    import numpy as np
    u8 = torch.arange(256, dtype=torch.uint8)
    want = torch.from_numpy(np.arange(256).astype(np.float32) / 255.0)
    assert torch.equal(u8.float() / 255.0, want)
    assert torch.equal(R.preprocess_u8(u8.view(1, 256, 1).expand(1, 256, 3)), E.bf(2.0 * want - 1.0).view(1, 256, 1)
                       .expand(1, 256, 3))


@pytest.mark.parametrize("use_eps", [True, False])
def test_preprocess_and_sample_pack_are_encode_images(use_eps):
    """vo.encode_images around a stub encoder: its input is the preprocess reference, its output the sample + pack"""
    h, w = 6, 10
    g = torch.Generator().manual_seed(7)
    img = torch.randint(0, 256, (8 * h, 8 * w, 3), generator=g, dtype=torch.uint8)
    lv = torch.linspace(-40, 30, h * w * 16).to(BF).view(h, w, 16)
    mean = (torch.randn(h, w, 16, generator=g) * 0.5).to(BF)
    eps = torch.randn(16, h, w, generator=g).to(BF) if use_eps else None
    stub = R.OracleStub(torch.cat([mean, lv], -1).permute(2, 0, 1)[None])
    want = vo.encode_images(stub, img, eps)[0]
    assert torch.equal(R.preprocess_u8(img), stub.seen[0].permute(1, 2, 0).float())
    mom = torch.cat([mean, lv, torch.zeros(h, w, 96, dtype=BF)], -1)
    assert torch.equal(R.sample_pack(mom, eps, shift=R.SHIFT_CPU), want.float())


# ------------------------------------------------------------------------------------ mutations
def _conv_fixture(H, W, stride, cfg, res, mut):
    x, w, b, r = G._operands(H, W, stride, cfg, res, True, "cpu")
    cout_pad = G.CONV_CFG[cfg][3]
    wf = torch.zeros(cout_pad, *w.shape[1:], dtype=BF)
    wf[:w.shape[0]] = w
    bf_ = torch.zeros(cout_pad, dtype=BF)
    bf_[:b.shape[0]] = b
    return R.conv(x, wf, bf_, stride, r), R.conv(x, wf, bf_, stride, r, mut=(mut,))


def _gn_fixture(H, W, C, seed, std, silu, mut):
    x, gamma, beta = G._gn_inputs(H, W, C, seed, std, device="cpu")
    return R.group_norm(x, gamma, beta, silu)[0], R.group_norm(x, gamma, beta, silu, mut=(mut,))[0]


def _sample_fixture(mut):
    """the eps case of test_sample_pack_logvar_sweep"""
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(BF)
    lv = bits[(bits.float() >= -40) & (bits.float() <= 30)]
    h = 2 * math.ceil(math.sqrt(lv.numel() / 16) / 2)
    w = 2 * math.ceil(lv.numel() / 16 / h / 2)
    g = torch.Generator().manual_seed(9)
    mom = torch.zeros(h, w, 128, dtype=BF)
    mom[..., 16:32] = torch.cat([lv, torch.zeros(h * w * 16 - lv.numel(), dtype=BF)]).view(h, w, 16)
    mom[: h // 2, :, :16] = (torch.randn(h // 2, w, 16, generator=g) * 0.5).to(BF)
    eps = torch.randn(16, h, w, generator=g).to(BF)
    return mom, eps, R.sample_pack(mom, eps), R.sample_pack(mom, eps, mut=(mut,))


def _mutated(mut):
    """(reference, mutated reference) on a fixture test_gpu_vae_ops.py runs (its seed where the seed matters)"""
    if mut == "s2_pad_topleft":
        return _conv_fixture(2, 2, 2, "c128", None, mut)
    if mut == "tap_corner":
        return _conv_fixture(6, 10, 1, "sc128_256", None, mut)
    if mut == "res_before_round":
        return _conv_fixture(6, 10, 1, "c256", "sep", mut)
    if mut == "gn_ring_count":
        return _gn_fixture(2, 2, 128, 128 + 7 * 2 + 2, 1.0, 0, mut)
    if mut == "gn_eps":
        return _gn_fixture(26, 22, 256, 5, 2.0 ** -6, 1, mut)
    if mut == "silu_unrounded":
        return _gn_fixture(6, 10, 256, 256 + 7 * 6 + 10, 1.0, 1, mut)
    if mut == "pad_keys_in":
        s = G._score_rows(128, 36, 128 + 36).float()
        return R.softmax_rows(s, 36)[:, :36], R.softmax_rows(s, 36, mut=(mut,))[:, :36]
    if mut in ("unpack_parity", "unpack_unrounded"):
        h = w = 64
        packed = _all_finite(h * w * 16)[torch.randperm(h * w * 16, generator=torch.Generator().manual_seed(0))]
        packed = packed.view((h // 2) * (w // 2), 64)
        return R.unpack_latents(packed, h, w), R.unpack_latents(packed, h, w, mut=(mut,))
    if mut == "upsample_round_up":
        x = E.randn((512, 512, 256), 2)
        return R.upsample2x(x), R.upsample2x(x, mut=(mut,))
    if mut in ("no_logvar_clamp", "shift_after_scale"):
        return _sample_fixture(mut)[2:]
    raise KeyError(mut)


@pytest.mark.parametrize("mut", sorted(R.MUTATIONS))
def test_mutation_is_caught(mut):
    ref, bad = _mutated(mut)
    frac = _changed(ref, bad)
    print(f"{mut}: {frac:.4f} of the outputs change")
    if mut == "no_logvar_clamp":
        # reachable: logvar > 20 (std e^10 against e^up-to-15).  Below -30 the std is < 2^-21 and the sample rounds
        # to the same bf16 value after the shift by 0.1159 either way.
        mom, eps, _, _ = _sample_fixture(mut)
        reach = R.pack(((mom[..., 16:32].float() > 20) & (eps.permute(1, 2, 0).float() != 0)).float()) > 0
        moved = ref.to(BF).view(torch.int16) != bad.to(BF).view(torch.int16)
        assert int(reach.sum()) > 0 and bool(moved[reach].all()) and not bool(moved[~reach].any())
    else:
        assert frac >= 0.01


# ------------------------------------------------------------------------------------ the binding
def test_hook_declarations_match_the_c_signatures():
    src = open(os.path.join(ROOT, "reflectionflow_b200", "csrc", "rf_api.cu")).read()
    kinds = {"int": "ci", "float": "cf"}
    for name, args in R.HOOKS.items():
        m = re.search(r"\bint " + name + r"\(([^)]*)\)", src)
        assert m, f"{name} is not defined in rf_api.cu"
        params = [p.strip() for p in m.group(1).replace("\n", " ").split(",") if p.strip() and p.strip() != "void"]
        got = [kinds.get(p.rsplit(" ", 1)[0].strip(), "vp") if "*" not in p else "vp" for p in params]
        assert got == args.split(), (name, got, args)
    header = open(os.path.join(ROOT, "include", "rf_b200.h")).read()
    assert "rf_dbg_vae" not in header  # test hooks stay out of the public ABI
