"""-m gpu: the VAE's kernels one launch at a time through the rf_dbg_vae_* hooks (csrc/rf_api.cu), which call the
launchers rf_vae_decode / rf_vae_encode run, against the references of tests/_vae_ref.py.

  * Convolution (conv_launch): bit-exact on exact operands for every pixel-tile width class of conv_tile_width, ragged
    and exact, stride 1 and 2, the real layers' channel counts (zero-padded ones included), residual separate and
    aliased with the output (the in-place conv_shortcut path of resnet()), with the one-pixel output ring and a guard
    region after the buffer unchanged.  The weight repack bit-exact against a permute + zero pad.  Random operands at
    K = 4608 to test_gpu_ops.py's GEMM bars.
  * GroupNorm (group_norm_launch): statistics (mean within 1e-6 of the group's RMS, 1 / std within 2^-12 relative)
    and outputs (<= 1 bf16 ulp, >= 99 % bit-identical) with a NaN input ring, both output layouts, large mean / std
    offsets, bit-identical reruns, and every finite bf16 value through the SiLU.
  * Row softmax with masked padding keys; the mid-block attention of both VAE halves through the real to_q | to_k |
    to_v stacking of rf_vae_load_weight; the layout kernels, bit-exact.

Measured on one H100 80GB HBM3 (700 W power limit), two runs with the same bits:
  convolution, repack, layout kernels   bit-exact everywhere
  GroupNorm                             1 / std within 2.2e-7 relative (also at mean / std = 128), mean within 6e-8 of
                                        the RMS; lowest bit-identical fraction 0.99998
  SiLU                                  0 ulps on all 65280 finite bf16 values (15569 in the flush band, all 0)
  softmax                               <= 1 ulp, lowest bit-identical fraction 0.99988
  mid-block attention                   |d| - 1 ulp <= 0.022 x RMS(to_out(O)); lowest bit-identical fraction 0.9749
                                        (decoder, 6 x 22); |ours - truth| = 0.88 ... 0.98 x |oracle bf16 - truth|: the
                                        bf16 scores cost nothing measurable against SDPA's own bf16 rounding points."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from reflectionflow_b200 import _lib as L  # noqa: E402
from tests import _exact as E  # noqa: E402
from tests import _vae_ref as R  # noqa: E402

DEV = "cuda:0"
BF = torch.bfloat16
SENT = 0x7FA5  # a NaN bit pattern no kernel writes: every element a launch must not touch holds it
GUARD = 4096


@pytest.fixture(scope="module")
def lib():
    return R.declare(L.load())


def _s():
    return L.cur_stream()


def _buf(n, dtype=BF):
    t = torch.empty(n + GUARD, dtype=dtype, device=DEV)
    (t.view(torch.int16) if dtype == BF else t).fill_(SENT if dtype == BF else 0xA5)
    return t


def _sent(t):
    return t.view(torch.int16) == SENT if t.dtype == BF else t == 0xA5


def _padded(buf, H, W, C):
    return buf[:(H + 2) * (W + 2) * C].view(H + 2, W + 2, C)


def _footprint(buf, H, W, C, chans=None, padded=True):
    """everything but the interior (its first `chans` channels) and the guard still holds the sentinel"""
    n = (H + 2) * (W + 2) * C if padded else H * W * C
    assert bool(_sent(buf[n:]).all()), "write past the end of the buffer"
    if padded:
        keep = torch.ones(H + 2, W + 2, C, dtype=torch.bool, device=DEV)
        keep[1:-1, 1:-1, :chans or C] = False
        assert bool(_sent(_padded(buf, H, W, C))[keep].all()), "write into the ring or the padding channels"


def _bits_equal(got, ref):
    return torch.equal(got.to(BF).view(torch.int16), ref.to(BF).view(torch.int16))


# ------------------------------------------------------------------------------------ convolution
def tile_width(H, W):
    """conv_tile_width (csrc/gemm_sm90.cu), restated to label the fixtures"""
    best, best_area = 128, None
    for bx in (128, 64, 32, 16, 8):
        area = -(-W // bx) * -(-H // (128 // bx))
        if best_area is None or area < best_area:
            best, best_area = bx, area
    return best


# name: (Cin real, Cin padded, Cout real, Cout padded, taps)
CONV_CFG = {
    "dec_conv_in": (16, 64, 512, 512, 9), "enc_conv_in": (3, 64, 128, 128, 9),
    "c128": (128, 128, 128, 128, 9), "c256": (256, 256, 256, 256, 9), "c512": (512, 512, 512, 512, 9),
    "sc512_256": (512, 512, 256, 256, 1), "sc128_256": (128, 128, 256, 256, 1),
    "dec_conv_out": (128, 128, 3, 128, 9), "enc_conv_out": (512, 512, 32, 128, 9),
}
# (output H, W, stride, layer, residual: None / "sep" / "alias"): the levels of 16^2, 208x176, 768x1344, 1360x768,
# 1008^2, 1024^2 and the 336x592 encode
CONV_CASES = [
    (2, 2, 1, "dec_conv_in", None), (2, 2, 1, "c128", "alias"), (2, 2, 1, "sc512_256", None),
    (2, 2, 1, "enc_conv_out", None),
    (6, 10, 1, "c256", "sep"), (6, 10, 1, "sc128_256", None), (6, 10, 1, "dec_conv_out", None),
    (6, 10, 1, "c512", "alias"),
    (26, 22, 1, "c512", None), (26, 22, 1, "enc_conv_in", None), (26, 22, 1, "sc512_256", "sep"),
    (96, 168, 1, "c256", "alias"), (96, 168, 1, "dec_conv_in", None),
    (170, 96, 1, "c128", "alias"), (170, 96, 1, "enc_conv_out", None),
    (126, 126, 1, "c512", "sep"), (126, 126, 1, "dec_conv_out", None),
    (128, 128, 1, "c512", "alias"), (128, 128, 1, "sc512_256", None),
    (1008, 1008, 1, "c128", "alias"), (1008, 1008, 1, "enc_conv_in", None),
    (2, 2, 2, "c128", None), (42, 74, 2, "c512", None), (84, 148, 2, "c256", None), (64, 64, 2, "c512", None),
]


def test_conv_fixtures_cover_every_tile_class():
    seen = {(tile_width(H, W), W % tile_width(H, W) != 0 or H % (128 // tile_width(H, W)) != 0, s)
            for H, W, s, _, _ in CONV_CASES}
    for bx, ragged in [(64, True), (16, True), (8, True), (8, False), (32, True), (128, True), (128, False),
                       (16, False)]:
        assert (bx, ragged, 1) in seen, (bx, ragged)
    assert {(16, True, 2), (32, True, 2), (64, True, 2)} <= seen  # 42x74, 84x148, 2x2
    assert {CONV_CFG[c][1:4:2] for _, _, _, c, _ in CONV_CASES} >= {(128, 128), (256, 256), (512, 512)}


def _operands(H, W, stride, cfg, res, exact, device=DEV):
    """(x, w, b, res) of a fixture, drawn on the CPU (the host tests draw the same ones)"""
    cin, cin_pad, cout, cout_pad, taps = CONV_CFG[cfg]
    k = 3 if taps == 9 else 1
    Hin, Win = stride * H, stride * W
    seed = H * 131 + W * 7 + stride
    if exact:
        x = E.act((Hin, Win, cin), seed)
        w = E.weight((cout, cin, k, k), seed + 1)
        b = E.weight((cout,), seed + 2)
        r = E.act((H, W, cout_pad), seed + 3) if res else None
    else:
        x = E.randn((Hin, Win, cin), seed)
        w = E.randn((cout, cin, k, k), seed + 1, 1.0 / math.sqrt(cin * k * k))
        b = E.randn((cout,), seed + 2, 0.05)
        r = E.randn((H, W, cout_pad), seed + 3) if res else None
    return tuple(None if t is None else t.to(device) for t in (x, w, b, r))


def _run_conv(lib, H, W, stride, cfg, res, x, w, b, r):
    cin, cin_pad, cout, cout_pad, taps = CONV_CFG[cfg]
    Hin, Win = stride * H, stride * W
    xp = torch.zeros(Hin + 2, Win + 2, cin_pad, dtype=BF, device=DEV)  # zero ring and zero padding channels
    xp[1:-1, 1:-1, :cin] = x
    nw = cout_pad * taps * cin_pad
    wr = _buf(nw)
    L.check(lib.rf_dbg_vae_conv_repack(R.ptr(w), R.ptr(wr), cout, cin, taps, cout_pad, cin_pad, _s()), "repack")
    bias = torch.zeros(cout_pad, dtype=BF, device=DEV)
    bias[:cout] = b
    ones = torch.ones(cout_pad, dtype=BF, device=DEV)
    out = _buf((H + 2) * (W + 2) * cout_pad)
    res_t = None
    if res == "alias":
        _padded(out, H, W, cout_pad)[1:-1, 1:-1] = r
        res_t = out
    elif res == "sep":
        res_t = R.pad(r)
    L.check(lib.rf_dbg_vae_conv(R.ptr(xp), R.ptr(wr), R.ptr(bias), R.ptr(out), R.ptr(res_t), R.ptr(ones), H, W,
                                cin_pad, cout_pad, taps, stride, _s()), "rf_dbg_vae_conv")
    torch.cuda.synchronize()
    return wr, nw, out


@pytest.mark.parametrize("H,W,stride,cfg,res", CONV_CASES)
def test_conv_bit_exact(lib, H, W, stride, cfg, res):
    cin, cin_pad, cout, cout_pad, taps = CONV_CFG[cfg]
    x, w, b, r = _operands(H, W, stride, cfg, res, True)
    wr, nw, out = _run_conv(lib, H, W, stride, cfg, res, x, w, b, r)
    assert _bits_equal(wr[:nw].view(cout_pad, -1), R.repack(w, cout_pad, cin_pad)), "weight repack"
    assert bool(_sent(wr[nw:]).all()), "repack wrote past its buffer"
    wf = torch.zeros(cout_pad, cin, w.shape[2], w.shape[3], dtype=BF, device=DEV)
    wf[:cout] = w
    bf_ = torch.zeros(cout_pad, dtype=BF, device=DEV)
    bf_[:cout] = b
    ref = R.conv(x, wf, bf_, stride, r)
    got = _padded(out, H, W, cout_pad)[1:-1, 1:-1]
    bad = (got.float() != ref).sum().item()
    assert bad == 0, f"{bad} of {ref.numel()} outputs differ"
    _footprint(out, H, W, cout_pad)


@pytest.mark.parametrize("H,W,stride,cfg,res", [(26, 22, 1, "c512", "alias"), (42, 74, 2, "c512", None),
                                                (6, 10, 1, "sc512_256", None)])
def test_conv_random_operands(lib, H, W, stride, cfg, res):
    """K = 4608 (and the 1x1 K = 512) with normal operands, held to test_gpu_ops.py's GEMM bars"""
    x, w, b, r = _operands(H, W, stride, cfg, res, False)
    _, _, out = _run_conv(lib, H, W, stride, cfg, res, x, w, b, r)
    ref = R.conv(x, w, b, stride, r, exact=False)
    got = _padded(out, H, W, CONV_CFG[cfg][3])[1:-1, 1:-1]
    torch.testing.assert_close(got.float(), ref, rtol=2 ** -7, atol=2e-2)
    _footprint(out, H, W, CONV_CFG[cfg][3])


def test_conv_refuses_unsupported_geometry(lib):
    z = torch.zeros(16, dtype=BF, device=DEV)
    for cin, cout, taps, stride in [(48, 128, 9, 1), (64, 96, 9, 1), (64, 128, 4, 1), (64, 128, 9, 3)]:
        assert lib.rf_dbg_vae_conv(R.ptr(z), R.ptr(z), R.ptr(z), R.ptr(z), None, R.ptr(z), 2, 2, cin, cout, taps,
                                   stride, _s()) == -1


# ------------------------------------------------------------------------------------ GroupNorm
GN_OUT_ULPS = 1
GN_FMA_SLACK = 2.0 ** -20  # 8 fp32 ulps of the larger summand
GN_IDENTICAL = 0.99
SILU_ARGMIN = -1.2784645  # SiLU's minimum, -0.2784645, is reached there
SILU_MIN = float(torch.tensor(-0.2784645).to(torch.bfloat16))


def _gn(lib, x, gamma, beta, silu, out_padded):
    H, W, C = x.shape
    xp = R.pad(x, float("nan"))  # production rings are zero: NaN proves they are never read
    n = (H + 2) * (W + 2) * C if out_padded else H * W * C
    out = _buf(n)
    part = torch.empty(lib.rf_dbg_vae_gn_part_floats(), dtype=torch.float32, device=DEV)
    mr = torch.full((64,), float("nan"), dtype=torch.float32, device=DEV)
    L.check(lib.rf_dbg_vae_group_norm(R.ptr(xp), R.ptr(out), H, W, C, R.ptr(gamma), R.ptr(beta), silu, 1, out_padded,
                                      R.ptr(part), R.ptr(mr), _s()), "rf_dbg_vae_group_norm")
    torch.cuda.synchronize()
    _footprint(out, H, W, C, padded=out_padded)
    got = _padded(out, H, W, C)[1:-1, 1:-1] if out_padded else out[:n].view(H, W, C)
    return got, mr


def _gn_inputs(H, W, C, seed, std=1.0, offset=0.0, device=DEV):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(H, W, C, generator=g) * std + offset).to(BF).to(device)
    gamma = (1 + 0.1 * torch.randn(C, generator=g)).to(BF).to(device)
    beta = (0.05 * torch.randn(C, generator=g)).to(BF).to(device)
    return x, gamma, beta


def _gn_check(lib, x, gamma, beta, silu, out_padded, tag):
    """statistics, then the normalised value y = bf16(t gamma + beta) within [lo, hi]: GN_OUT_ULPS bf16 ulps around the
    reference's value, widened by GN_FMA_SLACK (|t gamma| + |beta|) where the two summands cancel (a 1e-7 relative
    difference in t, the statistics' fp32 rounding, is many bf16 ulps of a y near 0).  With SiLU on, the output must lie
    in SiLU([lo, hi]): the SiLU of a bf16 value is exact (test_silu_every_bf16_value), and its slope times one ulp of y
    is several output ulps on its negative tail, so an ulp bar on the output would be looser there and tighter elsewhere
    than this one."""
    got, mr = _gn(lib, x, gamma, beta, silu, out_padded)
    pre, mean, rstd, terms = R.group_norm(x, gamma, beta, False, terms=True)
    C = x.shape[-1]
    rms = x.double().reshape(-1, 32, C // 32).pow(2).mean((0, 2)).sqrt()
    dm = ((mr[:32].double() - mean) / rms).abs().max().item()
    dr = (mr[32:].double() / rstd - 1).abs().max().item()
    slack = GN_FMA_SLACK * terms
    lo = R.bf16_step(E.bf(pre - slack), -GN_OUT_ULPS)
    hi = R.bf16_step(E.bf(pre + slack), GN_OUT_ULPS)
    if silu:
        a, b = R.silu(lo), R.silu(hi)
        low = torch.where((lo < SILU_ARGMIN) & (hi > SILU_ARGMIN), torch.full_like(a, SILU_MIN), torch.minimum(a, b))
        ok = (got.float() >= low) & (got.float() <= torch.maximum(a, b))
        same = _frac_equal(got, R.silu(pre))
    else:
        ok = (got.float() >= lo) & (got.float() <= hi)
        same = _frac_equal(got, pre)
    u = R.ulps(got, R.silu(pre) if silu else pre)
    print(f"[gn {tag}] |d mean| / rms {dm:.2e}  |d rstd| rel {dr:.2e}  max ulps {int(u.max())}  "
          f"outside [lo, hi] {int((~ok).sum())}  identical {same:.5f}")
    assert torch.isfinite(got.float()).all()
    assert dm <= 1e-6, f"group mean off by {dm:.3g} of the group's RMS"
    assert dr <= 2.0 ** -12, f"1 / std off by {dr:.3g} relative"
    assert bool(ok.all()) and same >= GN_IDENTICAL
    return got


def _frac_equal(got, ref):
    return (got.to(BF).view(torch.int16) == ref.to(BF).view(torch.int16)).double().mean().item()


@pytest.mark.parametrize("C", [128, 256, 512])
@pytest.mark.parametrize("H,W", [(2, 2), (6, 10), (26, 22), (128, 128)])
def test_group_norm(lib, C, H, W):
    x, gamma, beta = _gn_inputs(H, W, C, C + 7 * H + W)
    for silu in (0, 1):
        for out_padded in (1, 0):
            _gn_check(lib, x, gamma, beta, silu, out_padded, f"{H}x{W}x{C} silu {silu} padded out {out_padded}")


@pytest.mark.parametrize("H,W,C", [(1024, 1024, 128), (512, 512, 256)])
def test_group_norm_large_and_repeatable(lib, H, W, C):
    x, gamma, beta = _gn_inputs(H, W, C, 3)
    a = _gn_check(lib, x, gamma, beta, 1, 1, f"{H}x{W}x{C}")
    b, _ = _gn(lib, x, gamma, beta, 1, 1)
    assert _bits_equal(a, b), "two runs differ"


@pytest.mark.parametrize("ratio", [0, 8, 64, 128])
def test_group_norm_offset_mean(lib, ratio):
    """mean / std up to 128 at 1024^2 x 128 (std 0.5): E[x^2] - E[x]^2 from fp32 sums of x lost 2.9e-3 of 1 / std
    here; the statistics are now accumulated around a sample of each group"""
    x, gamma, beta = _gn_inputs(1024, 1024, 128, 11 + ratio, std=0.5, offset=0.5 * ratio)
    _gn_check(lib, x, gamma, beta, 1, 1, f"mean/std {ratio}")


def test_group_norm_small_variance(lib):
    """std 2^-6: eps = 1e-6 is a visible part of var + eps"""
    x, gamma, beta = _gn_inputs(26, 22, 256, 5, std=2.0 ** -6)
    _gn_check(lib, x, gamma, beta, 1, 1, "std 2^-6")


# SiLU's exemption: y < -126 ln 2 (about -87.34), where 1 + e^-y > 2^126 and __fdividef returns 0; the true value
# y e^y there is below 1e-36.
SILU_FLUSH_BELOW = -126 * math.log(2.0)


def test_silu_every_bf16_value(lib):
    """gamma = 0: the normalised value is exactly beta, so beta walks every finite bf16 value through the SiLU"""
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(BF)
    vals = bits[torch.isfinite(bits.float())]
    n = vals.numel()
    vals = torch.cat([vals, torch.zeros((-n) % 512, dtype=BF)]).to(DEV)
    x, _, _ = _gn_inputs(2, 2, 512, 1)
    gamma = torch.zeros(512, dtype=BF, device=DEV)
    worst, exempt = 0, 0
    for i in range(vals.numel() // 512):
        beta = vals[i * 512:(i + 1) * 512].contiguous()
        got, _ = _gn(lib, x, gamma, beta, 1, 0)
        ref = R.silu(beta.float())
        u = R.ulps(got, ref.expand_as(got))
        band = (beta.float() < SILU_FLUSH_BELOW).expand_as(got)
        exempt += int(band[0, 0].sum())
        assert (got.float()[band] == 0).all()
        worst = max(worst, int(u[~band].max()) if (~band).any() else 0)
    print(f"[silu] {n} finite bf16 values, max ulps {worst}, {exempt} in the flush band")
    assert worst <= 1


# ------------------------------------------------------------------------------------ row softmax
SM_IDENTICAL = 0.99


def _score_rows(n, valid, seed):
    """4 rows each of random, sharp (one key dominant), all-equal and |s| ~ 3000; padding keys large and finite"""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for kind in range(4):
        for _ in range(4):
            if kind == 0:
                r = torch.randn(n, generator=g) * 20
            elif kind == 1:
                r = torch.randn(n, generator=g) * 2
                r[torch.randint(0, valid, (1,), generator=g)] += 400
            elif kind == 2:
                r = torch.full((n,), 3.0)
            else:
                r = torch.sign(torch.randn(n, generator=g)) * 3000 + torch.randn(n, generator=g) * 40
            r[valid:] = 60000 * (1 + torch.rand(n - valid, generator=g))
            rows.append(r)
    return torch.stack(rows).to(BF)


@pytest.mark.parametrize("n", [128, 1024, 16384])
@pytest.mark.parametrize("dv", ["n", "n-1", "n-127", "4", "36"])
def test_softmax_rows(lib, n, dv):
    valid = {"n": n, "n-1": n - 1, "n-127": n - 127, "4": 4, "36": 36}[dv]
    s = _score_rows(n, valid, n + valid).to(DEV)
    ref = R.softmax_rows(s.float(), valid)
    got = s.clone()
    L.check(lib.rf_dbg_vae_softmax_rows(R.ptr(got), got.shape[0], n, valid, R.ATTN_SCALE_F32, _s()), "softmax")
    torch.cuda.synchronize()
    u = R.ulps(got[:, :valid], ref[:, :valid])
    same = (u == 0).double().mean().item()
    print(f"[softmax n {n} valid {valid}] max ulps {int(u.max())} identical {same:.5f}")
    assert int(u.max()) <= 1 and same >= SM_IDENTICAL
    assert bool((got[:, valid:].view(torch.int16) == 0).all()), "a padding key got a nonzero probability"


# ------------------------------------------------------------------------------------ mid-block attention
_MODELS = {}


def _vae():
    if not _MODELS:
        from oracle import vae_oracle as vo
        from reflectionflow_b200.vae import B200AutoencoderKL
        torch.manual_seed(0)
        ref = vo.AutoencoderKL()
        vo.init_weights_(ref, seed=0)
        ref.eval()
        _MODELS["m"] = (ref, B200AutoencoderKL().load_state_dict(ref.state_dict()))
    return _MODELS["m"]


# Bars of the kernel sequence against its float64 rounding-point reference, set on the first H100 run: S = q k^T is
# rounded to bf16 by both, but the GEMMs' fp32 sums and the reference's float64 ones land on different sides of a bf16
# midpoint now and then (|S| reaches ~100, where one bf16 ulp of S moves P by 2 %), and a moved S or P moves its whole
# output row a little.  The element bar is therefore 1 ulp of the output plus ATT_REL times the RMS of the attention
# branch to_out(O) of the row; the output itself is x + that branch, so an ulp bar alone fails where x + branch ~ 0.
ATT_REL = 2.0 ** -5
ATT_IDENTICAL = 0.97
ATT_TRUTH_MULT = 1.1  # |ours - truth| mean <= this x |oracle bf16 - truth| mean


@pytest.mark.parametrize("half", ["decoder", "encoder"])
@pytest.mark.parametrize("H,W", [(2, 2), (6, 6), (6, 22), (24, 40), (32, 32), (128, 128)])
def test_mid_attention(lib, half, H, W):
    ref_model, ours = _vae()
    att = getattr(ref_model, half).mid_block.attentions[0]
    p = {k: v.to(DEV) for k, v in att.state_dict().items()}
    g = torch.Generator().manual_seed(H * 1000 + W)
    x = torch.randn(H, W, 512, generator=g).to(BF).to(DEV)
    xp = R.pad(x, float("nan"))
    out = _buf((H + 2) * (W + 2) * 512)
    L.check(lib.rf_dbg_vae_mid_attention(ours._h, 1 if half == "encoder" else 0, R.ptr(xp), R.ptr(out), H, W, _s()),
            "rf_dbg_vae_mid_attention")
    torch.cuda.synchronize()
    _footprint(out, H, W, 512)
    got = _padded(out, H, W, 512)[1:-1, 1:-1].float()
    ref, branch = R.mid_attention(x, p)
    truth = R.mid_attention_truth(x, p)
    a16 = att.to(DEV)
    with torch.no_grad():
        o16 = a16(x.permute(2, 0, 1)[None].contiguous()).float()[0].permute(1, 2, 0)
    att.cpu()
    u = R.ulps(got, ref)
    same = (u == 0).double().mean().item()
    ulp = R.bf16_step(ref.abs(), 1) - ref.abs()
    scale = branch.double().pow(2).mean(-1, keepdim=True).sqrt()
    excess = (((got - ref).abs() - ulp).clamp(min=0).double() / scale).max().item()
    e_ours = (got.double() - truth).abs().mean().item()
    e_ref = (o16.double() - truth).abs().mean().item()
    e_kref = (ref.double() - truth).abs().mean().item()
    print(f"[mid attention {half} {H}x{W}] vs kernel-order ref: max (|d| - ulp) / rms(branch) {excess:.3e} "
          f"identical {same:.5f} ; "
          f"|ours-truth| {e_ours:.3e} |kernel-order ref-truth| {e_kref:.3e} |oracle bf16-truth| {e_ref:.3e} "
          f"(ratio {e_ours / e_ref:.3f})")
    assert torch.isfinite(got).all()
    assert excess <= ATT_REL and same >= ATT_IDENTICAL
    assert e_ours <= ATT_TRUTH_MULT * e_ref


# ------------------------------------------------------------------------------------ layout kernels
def _all_finite_bf16(n):
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(BF)
    v = bits[torch.isfinite(bits.float())]
    return torch.cat([v, torch.zeros(n - v.numel(), dtype=BF)])


def test_unpack_every_bf16_value(lib):
    h = w = 64  # 64 * 64 * 16 = 65536 latent values: every finite bf16 value once
    packed = _all_finite_bf16(h * w * 16)[torch.randperm(h * w * 16, generator=torch.Generator().manual_seed(0))]
    packed = packed.view((h // 2) * (w // 2), 64).to(DEV)
    out = _buf((h + 2) * (w + 2) * 64)
    L.check(lib.rf_dbg_vae_unpack_latents(R.ptr(packed), R.ptr(out), h, w, R.SCALING, R.SHIFT, _s()), "unpack")
    torch.cuda.synchronize()
    got = _padded(out, h, w, 64)[1:-1, 1:-1, :16]
    assert _bits_equal(got, R.unpack_latents(packed, h, w))
    _footprint(out, h, w, 64, chans=16)
    # the oracle's own decode_latents steps, run by torch on the GPU
    from oracle import vae_oracle as vo
    want = vo.decode_latents(R.OracleStub(), packed[None], 8 * h, 8 * w)[0].permute(1, 2, 0)
    assert _bits_equal(got, want)


def test_upsample_largest(lib):
    H, W, C = 512, 512, 256  # -> 1024^2 x 256, the decoder's largest tensor
    x = E.randn((H, W, C), 2, device=DEV)
    out = _buf((2 * H + 2) * (2 * W + 2) * C)
    L.check(lib.rf_dbg_vae_upsample2x(R.ptr(R.pad(x)), R.ptr(out), H, W, C, _s()), "upsample")
    torch.cuda.synchronize()
    assert _bits_equal(_padded(out, 2 * H, 2 * W, C)[1:-1, 1:-1], R.upsample2x(x))
    _footprint(out, 2 * H, 2 * W, C)


@pytest.mark.parametrize("H,W", [(6, 22), (128, 128)])
def test_repad_both_ways(lib, H, W):
    x = E.randn((H, W, 512), 3, device=DEV)
    comp = _buf(H * W * 512)
    L.check(lib.rf_dbg_vae_repad(R.ptr(R.pad(x, float("nan"))), R.ptr(comp), H, W, 512, 1, 0, _s()), "repad")
    back = _buf((H + 2) * (W + 2) * 512)
    L.check(lib.rf_dbg_vae_repad(R.ptr(comp), R.ptr(back), H, W, 512, 0, 1, _s()), "repad")
    torch.cuda.synchronize()
    assert _bits_equal(comp[:H * W * 512].view(H, W, 512), x)
    assert _bits_equal(_padded(back, H, W, 512)[1:-1, 1:-1], x)
    _footprint(comp, H, W, 512, padded=False)
    _footprint(back, H, W, 512)


def test_transpose_v(lib):
    npad = 16384
    qkv = E.randn((npad, 1536), 4, device=DEV)
    out = _buf(512 * npad)
    L.check(lib.rf_dbg_vae_transpose(R.ptr(qkv[:, 1024:]), 1536, R.ptr(out), npad, 512, _s()), "transpose")
    torch.cuda.synchronize()
    assert _bits_equal(out[:512 * npad].view(512, npad), qkv[:, 1024:].t())
    assert bool(_sent(out[512 * npad:]).all())


@pytest.mark.parametrize("src", ["u8", "chw"])
def test_image_to_nhwc(lib, src):
    H, W = 208, 176
    g = torch.Generator().manual_seed(5)
    img = torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8)
    img[0, :86, 0] = torch.arange(170, 256, dtype=torch.uint8)
    img[1, :170, 0] = torch.arange(0, 170, dtype=torch.uint8)  # every uint8 value
    chw = E.randn((3, H, W), 6, device=DEV)
    out = _buf((H + 2) * (W + 2) * 64)
    u8 = img.to(DEV)
    L.check(lib.rf_dbg_vae_image_to_nhwc(R.ptr(u8) if src == "u8" else None, R.ptr(chw) if src == "chw" else None,
                                         R.ptr(out), H, W, _s()), "image_to_nhwc")
    torch.cuda.synchronize()
    want = R.preprocess_u8(u8) if src == "u8" else chw.permute(1, 2, 0)
    assert _bits_equal(_padded(out, H, W, 64)[1:-1, 1:-1, :3], want)
    _footprint(out, H, W, 64, chans=3)


# bf16 logvar values where the device's expf and a correctly rounded exp round 0.5 logvar differently to bf16
# (none found on the H100; a value found later is listed here with its two results, not hidden by a looser bar)
EXP_DIFFERS = {}


@pytest.mark.parametrize("mode", ["eps", "mode"])
def test_sample_pack_logvar_sweep(lib, mode):
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(BF)
    lv = bits[(bits.float() >= -40) & (bits.float() <= 30)]
    h = 2 * math.ceil(math.sqrt(lv.numel() / 16) / 2)
    w = 2 * math.ceil(lv.numel() / 16 / h / 2)
    g = torch.Generator().manual_seed(9)
    mom = torch.zeros(h, w, 128, dtype=BF)
    flat = torch.cat([lv, torch.zeros(h * w * 16 - lv.numel(), dtype=BF)])
    mom[..., 16:32] = flat.view(h, w, 16)
    mom[: h // 2, :, :16] = (torch.randn(h // 2, w, 16, generator=g) * 0.5).to(BF)  # half the rows mean 0
    mom = mom.to(DEV)
    eps = torch.randn(16, h, w, generator=g).to(BF).to(DEV) if mode == "eps" else None
    out = _buf((h // 2) * (w // 2) * 64)
    L.check(lib.rf_dbg_vae_sample_pack(R.ptr(R.pad(mom, float("nan"))), 128, R.ptr(eps), R.ptr(out), h, w, R.SCALING,
                                       R.SHIFT, _s()), "sample_pack")
    torch.cuda.synchronize()
    n = (h // 2) * (w // 2) * 64
    got, ref = out[:n].view(-1, 64), R.sample_pack(mom, eps)
    diff = (got.view(torch.int16) != ref.to(BF).view(torch.int16))
    assert bool(_sent(out[n:]).all())
    assert int(diff.sum()) == 0, f"{int(diff.sum())} packed values differ"
    # the oracle's own encode_images steps after the encoder, run by torch on the GPU
    from oracle import vae_oracle as vo
    stub = R.OracleStub(mom[..., :32].permute(2, 0, 1)[None])
    want = vo.encode_images(stub, torch.zeros(8 * h, 8 * w, 3, dtype=torch.uint8, device=DEV), eps)[0]
    bad = (got.view(torch.int16) != want.view(torch.int16))
    assert int(bad.sum()) == 0, f"{int(bad.sum())} packed values differ from torch's evaluation of the oracle"


def test_postprocess_sweep(lib):
    """every bf16 value in [-1.5, 1.5] and +-inf to uint8 HWC (against the oracle's VaeImageProcessor) and bf16 CHW"""
    from oracle import vae_oracle as vo
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(BF)
    v = bits[(bits.float().abs() <= 1.5) | torch.isinf(bits.float())]
    H, W = 64, math.ceil(v.numel() / 3 / 64)
    flat = torch.cat([v, torch.zeros(H * W * 3 - v.numel(), dtype=BF)])
    img = flat.view(H, W, 3)
    x = torch.zeros(H, W, 128, dtype=BF)
    x[..., :3] = img
    x = x.to(DEV)
    u8 = _buf(H * W * 3, torch.uint8)
    chw = _buf(3 * H * W)
    L.check(lib.rf_dbg_vae_postprocess(R.ptr(R.pad(x, float("nan"))), H, W, 128, R.ptr(u8), R.ptr(chw), _s()),
            "postprocess")
    torch.cuda.synchronize()
    want = vo.postprocess_uint8(img.permute(2, 0, 1)[None])[0]
    assert torch.equal(u8[:H * W * 3].cpu().view(H, W, 3), want)
    assert _bits_equal(chw[:3 * H * W].view(3, H, W).cpu(), img.permute(2, 0, 1))
    assert bool(_sent(u8[H * W * 3:]).all()) and bool(_sent(chw[3 * H * W:]).all())
