"""References of the VAE's kernels (csrc/vae.cu and the convolution mode of csrc/gemm_sm90.cu), their named
mutations, and the ctypes binding of the test hooks that launch them (csrc/rf_api.cu: rf_dbg_vae_*).

Images are NHWC: a reference takes and returns the interior [H, W, C] as fp32 tensors holding bf16 values; the padded
layout of the kernels is [(H+2)(W+2), C] with a one-pixel ring (`pad` / `interior`).

  * Convolution: F.conv2d in float64 on the oracle's semantics (padding 1; stride 2 = diffusers Downsample2D's
    F.pad(x, (0, 1, 0, 1)) and no other padding), which knows nothing of the kernel's tap-major K or its TMA boxes.
    With operands on _exact.py's grids (activations k/8, weights and biases k/32) every partial sum is exact in fp32,
    so the kernel's accumulator is known exactly (`conv` asserts it) and the result is bit-exact.
  * GroupNorm(32, eps 1e-6): float64 statistics, then the kernel's formula bf16((x - mean) rstd gamma + beta) in fp32
    with its one fused multiply-add, then SiLU in float64 rounded to bf16.
  * Row softmax of bf16 scores with scale 1/sqrt(512) in float64 over the first `valid` keys; padding keys get 0.
  * Mid-block attention: `mid_attention` rounds to bf16 where the kernel sequence does (t, q | k | v, S = q k^T,
    P, O, the out-projection, the residual); `mid_attention_truth` is SDPA's semantics in float64.
  * Layout kernels as plain gathers and casts at the reference's rounding points: the latent unpack, nearest 2x,
    repad, transpose, VaeImageProcessor's pre- and post-process, the posterior sample + shift / scale + pack.

`mut` names one deliberate change from MUTATIONS; the host tests show each one moves a fixture the GPU tests run."""
import ctypes
import math
from ctypes import c_float, c_int, c_void_p

import torch
import torch.nn.functional as F

from oracle import vae_oracle as vo
from tests import _exact as E
from tests._exact import bf, f32

SCALING, SHIFT = vo.SCALING_FACTOR, vo.SHIFT_FACTOR
ATTN_SCALE = 1.0 / math.sqrt(512.0)
# the fp32 value the decoder passes to the softmax kernel: 1.0f / sqrtf(512.0f)
ATTN_SCALE_F32 = float(torch.tensor(1.0) / torch.sqrt(torch.tensor(512.0)))

MUTATIONS = {
    "s2_pad_topleft": "stride-2 convolution padded on the top / left instead of the bottom / right",
    "tap_corner": "1x1 convolution reads the tap at (0, 0) of the 3x3 window instead of the centre",
    "res_before_round": "residual added before the bias rounding: bf16(res + acc + bias)",
    "gn_ring_count": "GroupNorm statistics over the padded image (the zero ring counted)",
    "gn_eps": "GroupNorm eps 1e-5 instead of 1e-6",
    "silu_unrounded": "SiLU applied before the bf16 rounding of the normalised value",
    "pad_keys_in": "padding keys take part in the softmax",
    "unpack_parity": "latent unpack with the row / column parity bits swapped",
    "unpack_unrounded": "latent unpack without the bf16 rounding of z / scaling",
    "upsample_round_up": "nearest 2x reads source row (y + 1) >> 1",
    "no_logvar_clamp": "posterior sample without clamping logvar to [-30, 20]",
    "shift_after_scale": "(z * scale) - shift instead of (z - shift) * scale",
}


def pad(x, fill=0.0):
    """[H, W, C] -> [H+2, W+2, C] with the ring set to `fill`"""
    H, W, C = x.shape
    p = torch.full((H + 2, W + 2, C), fill, dtype=x.dtype, device=x.device)
    p[1:-1, 1:-1] = x
    return p


def interior(p):
    return p[1:-1, 1:-1]


def ulps(got, ref):
    return E.ulps(got, ref)


def bf16_step(t, k):
    """the bf16 value k steps from t along the bf16 number line"""
    b = t.to(torch.bfloat16).view(torch.int16).int()
    line = torch.where(b < 0, -(b & 0x7FFF), b) + k
    return torch.where(line < 0, (-line) | 0x8000, line).to(torch.int16).view(torch.bfloat16).float()


# ------------------------------------------------------------------------------------ convolution
def conv(x, w, b, stride=1, res=None, exact=True, mut=()):
    """x [Hin, Win, Cin] (interior), w [Cout, Cin, k, k] (torch layout), b [Cout], res [H, W, Cout] ->
    bf16(acc + b) or bf16(res + bf16(acc + b)), [H, W, Cout].  exact: assert that fp32 accumulation is exact."""
    xd = x.double().permute(2, 0, 1)[None]
    wd = w.double()

    def run(xx, ww):
        if w.shape[-1] == 1:
            if "tap_corner" in mut:
                xx = F.pad(xx, (1, 0, 1, 0))[..., :xx.shape[2], :xx.shape[3]]
            return F.conv2d(xx, ww)
        if stride == 2:
            return F.conv2d(F.pad(xx, (1, 0, 1, 0) if "s2_pad_topleft" in mut else (0, 1, 0, 1)), ww, stride=2)
        return F.conv2d(xx, ww, padding=1)

    y = run(xd, wd)
    if exact:
        e = E.lsb_exp(x) + E.lsb_exp(w)
        bound = run(xd.abs(), wd.abs()).max().item()
        assert bound < 2.0 ** (23 - e), f"operands not exact in fp32: sum |x w| = {bound} >= 2^{23 - e}"
        assert torch.equal(y.float().double(), y)
    acc = y[0].permute(1, 2, 0).float()
    v = acc + b.float()
    if res is None:
        return bf(v)
    if "res_before_round" in mut:
        return bf(res.float() + v)
    return bf(res.float() + bf(v))


def repack(w, cout_pad, cin_pad):
    """torch [Cout, Cin, k, k] -> [Cout_pad, k k Cin_pad], tap-major K, zero padded"""
    cout, cin, kh, kw = w.shape
    t = torch.zeros(cout_pad, kh, kw, cin_pad, dtype=w.dtype, device=w.device)
    t[:cout, :, :, :cin] = w.permute(0, 2, 3, 1)
    return t.reshape(cout_pad, kh * kw * cin_pad)


# ------------------------------------------------------------------------------------ GroupNorm
def gn_stats(x, mut=()):
    """float64 group mean and 1 / std of x [H, W, C] (32 groups)"""
    H, W, C = x.shape
    xg = x.double().reshape(H * W, 32, C // 32)
    if "gn_ring_count" in mut:
        n = (H + 2) * (W + 2) * (C // 32)
        mean = xg.sum((0, 2)) / n
        var = (xg * xg).sum((0, 2)) / n - mean * mean
    else:
        mean = xg.mean((0, 2))
        var = ((xg - mean[None, :, None]) ** 2).mean((0, 2))
    return mean, 1.0 / torch.sqrt(var + (1e-5 if "gn_eps" in mut else 1e-6))


def silu(v):
    d = v.double()
    return (d * torch.sigmoid(d)).to(torch.bfloat16).float()


def group_norm(x, gamma, beta, silu_on, mut=(), terms=False):
    """-> (out [H, W, C], mean [32] float64, rstd [32] float64) [, |t gamma| + |beta|: the size of the fused
    multiply-add's summands, which bounds its cancellation]"""
    C = x.shape[-1]
    mean, rstd = gn_stats(x, mut)
    mu = mean.float().repeat_interleave(C // 32)
    rs = rstd.float().repeat_interleave(C // 32)
    t = (x.float() - mu) * rs  # fp32, two roundings
    v = (t.double() * gamma.double() + beta.double()).float()  # the fused multiply-add: one rounding
    if silu_on and "silu_unrounded" in mut:
        return silu(v), mean, rstd
    y = bf(v)
    out = (silu(y) if silu_on else y), mean, rstd
    return out + ((t * gamma.float()).abs() + beta.float().abs(),) if terms else out


# ------------------------------------------------------------------------------------ attention
def softmax_rows(s, valid, scale=ATTN_SCALE, mut=()):
    """bf16(softmax(s * scale)) over keys [0, valid) of each row, 0 after"""
    d = s.double() * scale
    if "pad_keys_in" not in mut:
        d[:, valid:] = float("-inf")
    return bf(torch.softmax(d, dim=1).float())


def _lin(a, w, b):
    """bf16(a w^T + b): fp32 accumulation of bf16 operands, restated in float64"""
    return bf((a.double() @ w.double().t()).float() + b.float())


def mid_attention(x, p, mut=()):
    """the kernel sequence: x [H, W, 512] -> (out [H, W, 512], the attention branch to_out(O) [H, W, 512]); p: the
    VaeAttention's parameters (bf16) by name"""
    H, W, C = x.shape
    t, _, _ = group_norm(x, p["group_norm.weight"], p["group_norm.bias"], False, mut)
    t = t.reshape(H * W, C)
    q, k, v = (_lin(t, p[n + ".weight"], p[n + ".bias"]) for n in ("to_q", "to_k", "to_v"))
    S = bf((q.double() @ k.double().t()).float())
    P = softmax_rows(S, H * W, mut=mut)
    O = bf((P.double() @ v.double()).float())
    a = _lin(O, p["to_out.0.weight"], p["to_out.0.bias"])
    y = bf(x.reshape(H * W, C).float() + a)
    return y.reshape(H, W, C), a.reshape(H, W, C)


def mid_attention_truth(x, p):
    """SDPA's semantics in float64 (no rounding after the bf16 operands)"""
    H, W, C = x.shape
    xd = x.double().reshape(H * W, C)
    g = xd.reshape(H * W, 32, C // 32)
    mean = g.mean((0, 2), keepdim=True)
    var = ((g - mean) ** 2).mean((0, 2), keepdim=True)
    t = ((g - mean) / torch.sqrt(var + 1e-6)).reshape(H * W, C) * p["group_norm.weight"].double() \
        + p["group_norm.bias"].double()
    q, k, v = (t @ p[n + ".weight"].double().t() + p[n + ".bias"].double() for n in ("to_q", "to_k", "to_v"))
    o = torch.softmax((q @ k.t()) * ATTN_SCALE, dim=1) @ v
    y = xd + o @ p["to_out.0.weight"].double().t() + p["to_out.0.bias"].double()
    return y.reshape(H, W, C)


# ------------------------------------------------------------------------------------ layout kernels
# The shift is added to / subtracted from bf16 tensors as an fp32 scalar, as torch does on CUDA, where the reference
# pipeline runs.  torch on the CPU first rounds the scalar of a bf16 add / sub to bf16 (0.1159 -> 0.11572; its mul and
# div keep fp32): the host tests pass SHIFT_CPU to compare with the oracle run on the CPU.
SHIFT_CPU = float(torch.tensor(SHIFT).to(torch.bfloat16))


def unpack_latents(packed, h, w, mut=(), shift=SHIFT):
    """FluxPipeline._unpack_latents of [(h/2)(w/2), 64] -> z [h, w, 16], then bf16(bf16(z / scaling) + shift)"""
    z = packed.float().view(h // 2, w // 2, 16, 2, 2)
    z = z.permute(0, 4, 1, 3, 2) if "unpack_parity" in mut else z.permute(0, 3, 1, 4, 2)
    z = z.reshape(h, w, 16)
    q = z / f32(SCALING).to(z.device)
    if "unpack_unrounded" not in mut:
        q = bf(q)
    return bf(q + f32(shift).to(z.device))


def upsample2x(x, mut=()):
    """nearest 2x of [H, W, C]"""
    H, W, _ = x.shape
    ys = torch.arange(2 * H, device=x.device)
    ys = (ys + 1) >> 1 if "upsample_round_up" in mut else ys >> 1
    xs = torch.arange(2 * W, device=x.device) >> 1
    return pad(x)[ys + 1][:, xs + 1] if "upsample_round_up" in mut else x[ys][:, xs]


def preprocess_u8(img):
    """VaeImageProcessor.preprocess: uint8 [H, W, 3] -> bf16(2 (u8 / 255) - 1) in fp32, with numpy's (and torch's CPU)
    correctly rounded division; torch on CUDA divides by a scalar as a multiply by its reciprocal"""
    return bf(2.0 * (img.cpu().float() / 255.0) - 1.0).to(img.device)


def sample_pack(mom, eps=None, mut=(), shift=SHIFT):
    """moments [h, w, >= 32] (mean 0..15, logvar 16..31), eps [16, h, w] or None -> packed [(h/2)(w/2), 64]:
    DiagonalGaussianDistribution (logvar clamped, std = exp(0.5 logvar)) in bf16, then (z - shift) * scale, then
    FluxPipeline._pack_latents"""
    h, w, _ = mom.shape
    z = mom[..., :16].float()
    if eps is not None:
        lv = mom[..., 16:32].float()
        if "no_logvar_clamp" not in mut:
            lv = lv.clamp(-30.0, 20.0)
        sd = bf(torch.exp(bf(0.5 * lv).double()).float())
        z = bf(z + bf(sd * eps.float().permute(1, 2, 0)))
    sh, sc = f32(shift).to(z.device), f32(SCALING).to(z.device)
    z = bf(bf(z * sc) - sh) if "shift_after_scale" in mut else bf(bf(z - sh) * sc)
    return pack(z)


def pack(z):
    """FluxPipeline._pack_latents of [h, w, 16] -> [(h/2)(w/2), 64]"""
    h, w, _ = z.shape
    return z.reshape(h // 2, 2, w // 2, 2, 16).permute(0, 2, 4, 1, 3).reshape((h // 2) * (w // 2), 64)


class OracleStub:
    """an AutoencoderKL for oracle/vae_oracle.py's decode_latents / encode_images whose decoder is the identity and
    whose encoder returns given moments (and keeps its input): the oracle's own steps before and after the network"""

    def __init__(self, moments=None):
        self.moments, self.seen = moments, None

    def decode(self, z):
        return z

    def encoder(self, x):
        self.seen = x
        return self.moments

    encode_moments = vo.AutoencoderKL.encode_moments


# ------------------------------------------------------------------------------------ test-hook binding
HOOKS = {  # name -> argument types (vp: pointer, ci: int, cf: float)
    "rf_dbg_vae_conv": "vp vp vp vp vp vp ci ci ci ci ci ci vp",
    "rf_dbg_vae_conv_repack": "vp vp ci ci ci ci ci vp",
    "rf_dbg_vae_gn_part_floats": "",
    "rf_dbg_vae_group_norm": "vp vp ci ci ci vp vp ci ci ci vp vp vp",
    "rf_dbg_vae_mid_attention": "vp ci vp vp ci ci vp",
    "rf_dbg_vae_softmax_rows": "vp ci ci ci cf vp",
    "rf_dbg_vae_unpack_latents": "vp vp ci ci cf cf vp",
    "rf_dbg_vae_upsample2x": "vp vp ci ci ci vp",
    "rf_dbg_vae_repad": "vp vp ci ci ci ci ci vp",
    "rf_dbg_vae_transpose": "vp ci vp ci ci vp",
    "rf_dbg_vae_postprocess": "vp ci ci ci vp vp vp",
    "rf_dbg_vae_image_to_nhwc": "vp vp vp ci ci vp",
    "rf_dbg_vae_sample_pack": "vp ci vp vp ci ci cf cf vp",
}
_TYPES = {"vp": c_void_p, "ci": c_int, "cf": c_float}


def declare(lib):
    for name, args in HOOKS.items():
        fn = getattr(lib, name)
        fn.restype = c_int
        fn.argtypes = [_TYPES[a] for a in args.split()]
    return lib


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())
