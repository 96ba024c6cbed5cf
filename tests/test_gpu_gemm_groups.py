"""-m gpu: the grouped GEMM (csrc/gemm_sm90.cu) and the LoRA helper kernels at the operator level, through the test
hooks rf_dbg_* (csrc/rf_api.cu), in the launches enqueue_forward (csrc/dit.cu) makes:

  * up to three groups per launch with their own rows, weights, LoRA factors and per-section scales; fused LoRA
    groups, groups without a LoRA and groups under 128 rows that take the unfused `addend` (their term from an
    EPI_SCALE up-projection) in one launch; one and two 64-deep low-rank k-blocks (lora_pad 64 / 128);
  * bit-exact against tests/_exact.py on exact operands (every fp32 accumulator is known), the q|k|v epilogue
    (RMSNorm + RoPE) included, except the GELU epilogue (ex2.approx / rcp.approx against a float64 GELU: <= 1 ulp,
    >= 99.9 % identical, fp32 subnormals flushed to zero) and the grouped LayerNorm (its reduction order: the bars of
    test_gpu_ops.py::test_ln_modulate);
  * the same launches with random operands at the bars of test_gpu_ops.py;
  * an adapter with a different rank per module (peft rank_pattern) end to end against the CPU oracle."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from reflectionflow_b200 import _lib as L  # noqa: E402
from tests import _exact as E  # noqa: E402

DEV = "cuda:0"


@pytest.fixture(autouse=True)
def no_tf32():
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


@pytest.fixture(scope="module")
def lib():
    return E.declare(L.load())


@pytest.fixture(params=["pair", "single"])
def gemm_path(request, lib):
    """256-wide tiles where the launch picks them, and tiles at most 128 wide"""
    lib.rf_dbg_force_gemm_v1(1 if request.param == "single" else 0)
    yield request.param
    lib.rf_dbg_force_gemm_v1(0)


def _launch(lib, epi, N, K, groups):
    arr = E.groups_array(groups)
    L.check(lib.rf_dbg_gemm_grouped(epi, N, K, len(groups), arr, L.cur_stream()), "rf_dbg_gemm_grouped")
    torch.cuda.synchronize()


def _check(name, got, ref, how):
    got, ref = got.float(), ref.float()
    same = (got == ref).float().mean().item()
    u = E.ulps(got, ref)
    print(f"[{name}] identical {same:.5f} max ulps {u.max().item()} max |d| {(got - ref).abs().max().item():.4g}")
    assert torch.isfinite(got).all()
    if how == "exact":
        assert torch.equal(got, ref)
    elif how == "ulp":  # GELU: the kernel's ex2 / rcp flush fp32 subnormals to zero
        tiny = (ref.abs() < 2.0 ** -126) & (got.abs() < 2.0 ** -126)
        assert bool(((u <= 1) | tiny).all()) and same >= 0.999
    else:  # random operands: test_gpu_ops.py's bars
        torch.testing.assert_close(got, ref, rtol=2 ** -6, atol=3e-2)
        assert same >= 0.98


# ------------------------------------------------------------------------------------ operands
def _x(M, K, seed, exact):
    return E.act((M, K), seed, DEV) if exact else E.randn((M, K), seed, 1.0, DEV)


def _w(N, K, seed, exact):
    return E.weight((N, K), seed, DEV) if exact else E.randn((N, K), seed, 1 / math.sqrt(K), DEV)


def _factors(K, N, nsec, pad, rank, seed, exact):
    """stacked zero-padded factors of nsec targets: A_all [nsec pad, K], B_all [N, pad]"""
    A = torch.zeros(nsec * pad, K, dtype=torch.bfloat16, device=DEV)
    B = torch.zeros(N, pad, dtype=torch.bfloat16, device=DEV)
    w = N // nsec
    for s in range(nsec):
        if exact:
            A[s * pad:s * pad + rank] = E.weight((rank, K), seed + s, DEV)
            B[s * w:(s + 1) * w, :rank] = E.lora_b((w, rank), seed + 10 + s, DEV)
        else:
            A[s * pad:s * pad + rank] = E.randn((rank, K), seed + s, 1 / math.sqrt(K), DEV)
            B[s * w:(s + 1) * w, :rank] = E.randn((w, rank), seed + 10 + s, 0.5 / math.sqrt(rank), DEV)
    return A, B


def _rope(M, seed):
    g = torch.Generator().manual_seed(seed)
    ang = torch.rand(M, 64, generator=g) * 6.28
    return ang.cos().contiguous().to(DEV), ang.sin().contiguous().to(DEV)


def _norm_w(seed):
    return (1.0 + 0.1 * E.randn((128,), seed, 1.0, DEV).float()).to(torch.bfloat16)


class Stream:
    """one token stream (group) of a launch: rows x [M, K] (a view into an A buffer of pitch a_pitch at column a_off),
    its weights, an optional LoRA (A_all, B_all, scales), and the output view"""

    def __init__(self, M, K, N, seed, exact, W, bias, lora=None, a_pitch=None, a_off=0):
        buf = _x(M, a_pitch or K, seed, exact)
        self.x = buf[:, a_off:a_off + K]
        self.W, self.bias, self.lora, self.M, self.N, self.K = W, bias, lora, M, N, K


def _run_launch(lib, epi, streams, pad, sec_cols, exact, out_pitch=None, out_off=0, heads=None, seed=0,
                res_pitch=None):
    """Launch `streams` as one grouped GEMM the way project() in csrc/dit.cu does (fused LoRA groups of >= 128
    rows, the unfused EPI_SCALE term into an addend below) and return [(got, ref)] per stream."""
    N, K = streams[0].N, streams[0].K
    nsec = N // sec_cols if sec_cols else 1
    groups, outs, refs, keep = [], [], [], []
    for j, st in enumerate(streams):
        kw = {}
        L_ref = None
        if st.lora is not None:
            A_all, B_all, scales = st.lora
            T = E.lora_down(st.x, A_all, exact).to(torch.bfloat16)
            L_ref = E.lora_up(T.float(), B_all, scales, sec_cols, pad, exact)
            if st.M >= 128:
                kw.update(T=T, B=B_all, sec_cols=sec_cols, pad=pad, scales=scales)
            else:  # lora_term: one EPI_SCALE group per section into the addend
                Lb = torch.full((st.M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
                w = N // nsec
                ug = [E.group(T[:, s * pad:(s + 1) * pad], B_all[s * w:(s + 1) * w], Lb[:, s * w:(s + 1) * w],
                              scales=(scales[s],)) for s in range(nsec)]
                _launch(lib, E.EPI_SCALE, w, pad, ug)
                _check(f"stream {j} unfused term", Lb, L_ref, "exact" if exact else "rand")
                kw["addend"] = Lb
            keep.append(T)
        if epi == E.EPI_GATE_RES:
            X = E.randn((st.M, res_pitch or N), seed + 50 + j, 1.0, DEV)
            out = X[:, :N]
            res0 = out.clone()
            gate = E.randn((N,), seed + 60 + j, 0.5, DEV)
            kw.update(res=out, gate=gate)
            keep += [X, gate]
        else:
            buf = torch.full((st.M, out_pitch or N), float("nan"), dtype=torch.bfloat16, device=DEV)
            out = buf[:, out_off:out_off + N]
            keep.append(buf)
        if epi == E.EPI_QKV:
            cos, sin = _rope(st.M, seed + 70 + j)
            nq, nk = _norm_w(seed + 80 + j), _norm_w(seed + 90 + j)
            kw.update(cos=cos, sin=sin, nq=nq, nk=nk)
            keep += [cos, sin, nq, nk]
        groups.append(E.group(st.x, st.W, out, bias=st.bias, **kw))
        v = E.linear(st.x, st.W, st.bias, L=L_ref, exact=exact)
        if epi == E.EPI_GATE_RES:
            ref = E.gate_res(v, res0, kw["gate"])
        elif epi == E.EPI_GELU:
            ref = E.gelu(v)
        elif epi == E.EPI_QKV:
            ref = E.qkv_post(v, kw["cos"], kw["sin"], kw["nq"], kw["nk"], heads)
        else:
            ref = v
        outs.append(out)
        refs.append(ref)
    _launch(lib, epi, N, K, groups)
    return list(zip(outs, refs))


def _qkv_streams(rows, heads, K, pad, rank, scales, exact, seed=0, lora_on=(True, True, True)):
    """[txt, img, cond] in enqueue_forward's group order (img, txt, cond): text weights / factors for txt, shared ones
    for img and cond"""
    D = heads * 128
    N = 3 * D
    Wt, Ws = _w(N, K, seed + 1, exact), _w(N, K, seed + 2, exact)
    bt, bs = E.randn((N,), seed + 3, 0.5, DEV), E.randn((N,), seed + 4, 0.5, DEV)
    At, Bt = _factors(K, N, 3, pad, rank, seed + 100, exact)
    As, Bs = _factors(K, N, 3, pad, rank, seed + 200, exact)
    m_txt, m_img, m_cond = rows
    return [Stream(m_img, K, N, seed + 5, exact, Ws, bs, (As, Bs, scales[1]) if lora_on[1] else None),
            Stream(m_txt, K, N, seed + 6, exact, Wt, bt, (At, Bt, scales[0]) if lora_on[0] else None),
            Stream(m_cond, K, N, seed + 7, exact, Ws, bs, (As, Bs, scales[2]) if lora_on[2] else None)]


QKV_SCALES = ((0.5, 1.0, -0.75), (2.0, 0.25, 1.0), (-1 / 3, 0.75, 1.5))  # txt, img, cond; sections q, k, v


# ------------------------------------------------------------------------------------ q|k|v
@pytest.mark.parametrize("pad,rank", [(64, 64), (128, 96)])
def test_double_block_qkv_headline_exact(lib, pad, rank):
    """txt 512 + img 4096 + cond 1024 rows, N = 9216, K = 3072, BN = 256; every group fused, scales per section and
    per group"""
    streams = _qkv_streams((512, 4096, 1024), 24, 3072, pad, rank, QKV_SCALES, True)
    for j, (got, ref) in enumerate(_run_launch(lib, E.EPI_QKV, streams, pad, 3072, True, heads=24)):
        _check(f"qkv headline pad {pad} group {j}", got, ref, "exact")


@pytest.mark.parametrize("heads", [24, 3])
def test_qkv_ragged_groups_exact(lib, heads, gemm_path):
    """txt 77 (unfused: EPI_SCALE term into an addend), img 1000, cond 576 (a 384x384 condition); heads = 3 puts
    384-column sections under 128-wide tiles"""
    pad = 128 if heads == 3 else 64
    streams = _qkv_streams((77, 1000, 576), heads, 1024, pad, pad, QKV_SCALES, True, seed=11)
    for j, (got, ref) in enumerate(_run_launch(lib, E.EPI_QKV, streams, pad, heads * 128, True, heads=heads)):
        _check(f"qkv ragged h{heads} group {j}", got, ref, "exact")


@pytest.mark.parametrize("case", ["headline", "ragged"])
def test_qkv_random_operands(lib, case):
    if case == "headline":
        rows, heads, K, pad, rank = (512, 4096, 1024), 24, 3072, 128, 128
    else:
        rows, heads, K, pad, rank = (77, 1000, 576), 3, 1024, 64, 32
    streams = _qkv_streams(rows, heads, K, pad, rank, QKV_SCALES, False, seed=21)
    for j, (got, ref) in enumerate(_run_launch(lib, E.EPI_QKV, streams, pad, heads * 128, False, heads=heads)):
        _check(f"qkv random {case} group {j}", got, ref, "rand")


def test_qkv_mixed_lora_and_plain_groups(lib, gemm_path):
    """img without a LoRA, txt fused, cond 64 rows unfused, in one launch"""
    streams = _qkv_streams((256, 384, 64), 2, 512, 64, 48, QKV_SCALES, True, seed=31, lora_on=(True, False, True))
    for j, (got, ref) in enumerate(_run_launch(lib, E.EPI_QKV, streams, 64, 256, True, heads=2)):
        _check(f"qkv mixed group {j}", got, ref, "exact")


# ------------------------------------------------------------------------------------ scale edges
def test_section_scale_edges(lib):
    """s = (1, 1, 1) equals the op that applies no scaling (rf_op_linear_lora) bit for bit; s = 0 on section k only
    leaves that section equal to the adapter-free output; negative and 1/3 scales match the reference"""
    heads, K, pad = 2, 512, 64
    D = heads * 128
    outs = {}
    for tag, sc in (("one", (1.0, 1.0, 1.0)), ("zero_k", (-0.75, 0.0, 1 / 3)), ("none", None)):
        st = _qkv_streams((0, 384, 0), heads, K, pad, 32, (sc or (1, 1, 1),) * 3, True, seed=41,
                          lora_on=(False, sc is not None, False))[0]
        (got, ref), = _run_launch(lib, E.EPI_QKV, [st], pad, D, True, heads=heads, seed=41)
        _check(f"scale edge {tag}", got, ref, "exact")
        outs[tag] = (got.clone(), st)
    # the zero section equals the adapter-free output, the others do not
    z, free = outs["zero_k"][0], outs["none"][0]
    assert torch.equal(z[:, D:2 * D], free[:, D:2 * D])
    assert not torch.equal(z[:, :D], free[:, :D]) and not torch.equal(z[:, 2 * D:], free[:, 2 * D:])
    # unit scales: the same bits as the ABI op, which runs the fused LoRA without a scale
    got1, st = outs["one"]
    A_all, B_all, _ = st.lora
    y = torch.empty_like(got1)
    cos, sin = _rope(st.M, 41 + 70)
    nq, nk = _norm_w(41 + 80), _norm_w(41 + 90)
    ws = torch.zeros(lib.rf_op_linear_lora_workspace_bytes(st.M), dtype=torch.uint8, device=DEV)
    rc = lib.rf_op_linear_lora(E.EPI_QKV, st.M, 3 * D, K, L.ptr(st.x), st.x.stride(0), L.ptr(st.W), L.ptr(st.bias),
                               L.ptr(y), y.stride(0), L.ptr(A_all), 192, L.ptr(B_all), None, 0, None, L.ptr(cos),
                               L.ptr(sin), L.ptr(nq), L.ptr(nk), L.ptr(ws), L.cur_stream())
    L.check(rc, "rf_op_linear_lora")
    torch.cuda.synchronize()
    assert torch.equal(y, got1)


# ------------------------------------------------------------------------------------ to_out / ff.net.2 / proj_out
@pytest.mark.parametrize("which,K,off", [("to_out", 3072, 0), ("ff.net.2", 12288, 3072), ("proj_out", 15360, 0)])
def test_gate_res_in_place_exact(lib, which, K, off):
    """GATE_RES in place on X (D = 3072), A read from the 5D-pitched ACT buffer: img 1024 fused (shared factors),
    txt 512 fused (text factors, two k-blocks), cond 77 unfused"""
    D = 3072
    Ws, Wt = _w(D, K, 1, True), _w(D, K, 2, True)
    bs, bt = E.randn((D,), 3, 0.5, DEV), E.randn((D,), 4, 0.5, DEV)
    As, Bs = _factors(K, D, 1, 128, 128, 300, True)
    At, Bt = _factors(K, D, 1, 128, 80, 400, True)
    streams = [Stream(1024, K, D, 5, True, Ws, bs, (As, Bs, (-0.75,)), a_pitch=5 * D, a_off=off),
               Stream(512, K, D, 6, True, Wt, bt, (At, Bt, (1 / 3,)), a_pitch=5 * D, a_off=off),
               Stream(77, K, D, 7, True, Ws, bs, (As, Bs, (-0.75,)), a_pitch=5 * D, a_off=off)]
    for j, (got, ref) in enumerate(_run_launch(lib, E.EPI_GATE_RES, streams, 128, 0, True)):
        _check(f"{which} group {j}", got, ref, "exact")


def test_gate_res_random_operands(lib):
    D, K = 3072, 3072
    W, bias = _w(D, K, 1, False), E.randn((D,), 3, 0.1, DEV)
    A, B = _factors(K, D, 1, 64, 32, 300, False)
    streams = [Stream(1000, K, D, 5, False, W, bias, (A, B, (0.8,)), a_pitch=5 * D),
               Stream(77, K, D, 7, False, W, bias, (A, B, (0.8,)), a_pitch=5 * D)]
    for j, (got, ref) in enumerate(_run_launch(lib, E.EPI_GATE_RES, streams, 64, 0, False)):
        _check(f"gate_res random group {j}", got, ref, "rand")


@pytest.mark.parametrize("N", [1664, 3584])
def test_decode_remainder_band(lib, N):
    """more than 12 n-tiles, not a multiple of the band of 4 (13 tiles at BN 128, 14 at BN 256): the remainder branch
    of decode_tile with several groups"""
    K = 512
    W, bias = _w(N, K, 1, True), E.randn((N,), 3, 0.5, DEV)
    A, B = _factors(K, N, 1, 64, 64, 300, True)
    streams = [Stream(300, K, N, 5, True, W, bias, (A, B, (1 / 3,))),
               Stream(129, K, N, 6, True, W, bias, None),
               Stream(640, K, N, 7, True, W, bias, (A, B, (-0.75,)))]
    for j, (got, ref) in enumerate(_run_launch(lib, E.EPI_GATE_RES, streams, 64, 0, True)):
        _check(f"decode N={N} group {j}", got, ref, "exact")


# ------------------------------------------------------------------------------------ MLP-in (GELU)
def test_mlp_in_gelu(lib, gemm_path):
    """GELU into columns [D, 5D) of a 5D-pitched buffer (D = 256): img fused, txt plain, cond 64 unfused"""
    D, K, N = 256, 256, 1024
    W, bias = _w(N, K, 1, True), E.randn((N,), 3, 0.5, DEV)
    A, B = _factors(K, N, 1, 128, 128, 300, True)
    streams = [Stream(512, K, N, 5, True, W, bias, (A, B, (1 / 3,))),
               Stream(128, K, N, 6, True, _w(N, K, 2, True), bias, None),
               Stream(64, K, N, 7, True, W, bias, (A, B, (1 / 3,)))]
    for j, (got, ref) in enumerate(_run_launch(lib, E.EPI_GELU, streams, 128, 0, True, out_pitch=5 * D,
                                               out_off=D)):
        _check(f"mlp-in gelu group {j}", got, ref, "ulp")


# ------------------------------------------------------------------------------------ single block's shared T
@pytest.mark.parametrize("lpad", [64, 128])
def test_single_block_shared_T(lib, lpad):
    """T for to_q|to_k|to_v|proj_mlp of all LoRA'd rows in one grouped lora_down (NT = 4 lpad): the txt + img rows
    contiguous with the shared factors as one group (project() merges such runs), the cond rows with a second factor
    set; then the q|k|v launch reads T at pitch 4 lpad and the GELU launch at column 3 lpad."""
    heads, D = 2, 256
    n_main, n_cond = 640, 192
    XN = E.act((n_main + n_cond, D), 1, DEV)
    A4 = E.weight((4 * lpad, D), 2, DEV)
    A4c = E.weight((4 * lpad, D), 3, DEV)
    T = torch.full((n_main + n_cond, 4 * lpad), float("nan"), dtype=torch.bfloat16, device=DEV)
    dg = [E.group(XN[:n_main], A4, T[:n_main]), E.group(XN[n_main:], A4c, T[n_main:])]
    arr = E.groups_array(dg)
    L.check(lib.rf_dbg_lora_down_grouped(D, 4 * lpad, 2, arr, L.cur_stream()), "rf_dbg_lora_down_grouped")
    torch.cuda.synchronize()
    T_ref = torch.cat([E.lora_down(XN[:n_main], A4), E.lora_down(XN[n_main:], A4c)])
    _check("lora_down grouped", T, T_ref, "exact")
    Tf = T_ref
    # q|k|v: B [3D, lpad], T columns [lpad s, lpad (s + 1)) of pitch 4 lpad
    Bq, Bqc = E.lora_b((3 * D, lpad), 4, DEV), E.lora_b((3 * D, lpad), 5, DEV)
    Wq, bq = E.weight((3 * D, D), 6, DEV), E.randn((3 * D,), 7, 0.5, DEV)
    sc, scc = (0.5, -0.75, 1 / 3), (1.5, 1.0, -2.0)
    qkv = torch.full((n_main + n_cond, 3 * D), float("nan"), dtype=torch.bfloat16, device=DEV)
    cos, sin = _rope(n_main + n_cond, 8)
    nq, nk = _norm_w(9), _norm_w(10)
    g = [E.group(XN[:n_main], Wq, qkv[:n_main], bias=bq, cos=cos[:n_main], sin=sin[:n_main], nq=nq, nk=nk,
                 T=T[:n_main], B=Bq, sec_cols=D, pad=lpad, scales=sc),
         E.group(XN[n_main:], Wq, qkv[n_main:], bias=bq, cos=cos[n_main:], sin=sin[n_main:], nq=nq, nk=nk,
                 T=T[n_main:], B=Bqc, sec_cols=D, pad=lpad, scales=scc)]
    _launch(lib, E.EPI_QKV, 3 * D, D, g)
    for r, Bx, s in ((slice(0, n_main), Bq, sc), (slice(n_main, None), Bqc, scc)):
        Lr = E.lora_up(Tf[r, :3 * lpad], Bx, s, D, lpad)
        ref = E.qkv_post(E.linear(XN[r], Wq, bq, L=Lr), cos[r], sin[r], nq, nk, heads)
        _check(f"shared T qkv rows {r}", qkv[r], ref, "exact")
    # proj_mlp: T columns [3 lpad, 4 lpad)
    Bm, Bmc = E.lora_b((4 * D, lpad), 11, DEV), E.lora_b((4 * D, lpad), 12, DEV)
    Wm, bm = E.weight((4 * D, D), 13, DEV), E.randn((4 * D,), 14, 0.5, DEV)
    act = torch.full((n_main + n_cond, 5 * D), float("nan"), dtype=torch.bfloat16, device=DEV)
    g = [E.group(XN[:n_main], Wm, act[:n_main, D:], bias=bm, T=T[:n_main, 3 * lpad:], B=Bm, pad=lpad,
                 scales=(-0.75,)),
         E.group(XN[n_main:], Wm, act[n_main:, D:], bias=bm, T=T[n_main:, 3 * lpad:], B=Bmc, pad=lpad,
                 scales=(1 / 3,))]
    _launch(lib, E.EPI_GELU, 4 * D, D, g)
    for r, Bx, s in ((slice(0, n_main), Bm, -0.75), (slice(n_main, None), Bmc, 1 / 3)):
        Lr = E.lora_up(Tf[r, 3 * lpad:], Bx, (s,), 0, lpad)
        _check(f"shared T mlp rows {r}", act[r, D:], E.gelu(E.linear(XN[r], Wm, bm, L=Lr)), "ulp")


# ------------------------------------------------------------------------------------ EPI_SCALE / EPI_BIAS
@pytest.mark.parametrize("lpad", [64, 128])
def test_scale_up_projection_exact(lib, lpad, gemm_path):
    """lora_term's up-projection: three groups (q, k, v) with their own scales, output pitch 3D; and the final
    proj_out's N = 64 (BN = 64)"""
    D, M = 3072, 77
    T = E.lora_down(E.act((M, 512), 1, DEV), E.weight((3 * lpad, 512), 2, DEV)).to(torch.bfloat16)
    Bs = [E.lora_b((D, lpad), 3 + s, DEV) for s in range(3)]
    Lb = torch.full((M, 3 * D), float("nan"), dtype=torch.bfloat16, device=DEV)
    sc = (-0.75, 1 / 3, 2.0)
    g = [E.group(T[:, s * lpad:(s + 1) * lpad], Bs[s], Lb[:, s * D:(s + 1) * D], scales=(sc[s],)) for s in range(3)]
    _launch(lib, E.EPI_SCALE, D, lpad, g)
    for s in range(3):
        ref = E.scale_out(E.linear(T[:, s * lpad:(s + 1) * lpad], Bs[s]), sc[s])
        _check(f"EPI_SCALE section {s}", Lb[:, s * D:(s + 1) * D], ref, "exact")
    B64 = E.lora_b((64, lpad), 9, DEV)
    L64 = torch.full((M, 64), float("nan"), dtype=torch.bfloat16, device=DEV)
    _launch(lib, E.EPI_SCALE, 64, lpad, [E.group(T[:, :lpad], B64, L64, scales=(1 / 3,))])
    _check("EPI_SCALE N=64", L64, E.scale_out(E.linear(T[:, :lpad], B64), 1 / 3), "exact")


def test_bias_grouped_with_addend_exact(lib, gemm_path):
    """EPI_BIAS over three ragged groups (the embedders' launch), one with an addend"""
    N, K = 3072, 64
    W, bias = _w(N, K, 1, True), E.randn((N,), 2, 0.5, DEV)
    xs = [E.act((m, K), 3 + i, DEV) for i, m in enumerate((1000, 576, 77))]
    add = E.randn((576, N), 9, 1.0, DEV)
    outs = [torch.full((x.shape[0], N), float("nan"), dtype=torch.bfloat16, device=DEV) for x in xs]
    g = [E.group(xs[0], W, outs[0], bias=bias), E.group(xs[1], W, outs[1], bias=bias, addend=add),
         E.group(xs[2], W, outs[2], bias=bias)]
    _launch(lib, E.EPI_BIAS, N, K, g)
    for j, x in enumerate(xs):
        _check(f"bias group {j}", outs[j], E.linear(x, W, bias, addend=add if j == 1 else None), "exact")


# ------------------------------------------------------------------------------------ helper kernels
def test_add_rows_exact(lib):
    """the adaLN / embedder LoRA add: dst[b, sec] = bf16(dst + bf16(src * s)) on a strided row set"""
    rows, cols, ld = 3, 6 * 3072, 20000
    dst = E.randn((rows, ld), 1, 1.0, DEV)
    src = E.lora_down(E.act((rows, 256), 2, DEV), E.weight((cols, 256), 3, DEV)).to(torch.bfloat16)
    for s in (1 / 3, -0.75):
        d = dst.clone()
        L.check(lib.rf_dbg_add_rows(d.data_ptr(), ld, src.data_ptr(), cols, rows, cols, s, L.cur_stream()),
                "rf_dbg_add_rows")
        torch.cuda.synchronize()
        _check(f"add_rows s={s:.4g}", d[:, :cols], E.add_rows(dst[:, :cols], src, s), "exact")
        assert torch.equal(d[:, cols:], dst[:, cols:])


@pytest.mark.parametrize("R", [64, 128])
def test_lora_merge_exact(lib, R):
    N, K = 384, 3072
    W = E.act((N, K), 1, DEV)
    A = E.dyadic((R, K), 6, 64, 2, DEV)
    B = E.weight((N, R), 3, DEV)
    for s in (1 / 3, -0.75):
        Wm = torch.full_like(W, float("nan"))
        L.check(lib.rf_dbg_lora_merge(W.data_ptr(), A.data_ptr(), B.data_ptr(), Wm.data_ptr(), N, K, R, s,
                                      L.cur_stream()), "rf_dbg_lora_merge")
        torch.cuda.synchronize()
        _check(f"lora_merge R={R} s={s:.4g}", Wm, E.lora_merge(W, A, B, s), "exact")


def test_ln_modulate_grouped(lib):
    """three row ranges of one buffer with their own (scale, shift): the bars of test_gpu_ops.py::test_ln_modulate"""
    dim, ends = 3072, (77, 1077, 1653)
    x = E.randn((ends[-1], dim), 1, 3.0, DEV) + 0.5
    sc = [E.randn((dim,), 2 + i, 0.3, DEV) for i in range(3)]
    sh = [E.randn((dim,), 5 + i, 0.3, DEV) for i in range(3)]
    out = torch.full_like(x, float("nan"))
    row_end = (ctypes.c_int * 3)(*ends)
    scp = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in sc])
    shp = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in sh])
    L.check(lib.rf_dbg_ln_modulate_grouped(x.data_ptr(), dim, out.data_ptr(), dim, dim, 3, row_end, scp, shp,
                                           L.cur_stream()), "rf_dbg_ln_modulate_grouped")
    torch.cuda.synchronize()
    ln = E.bf(F.layer_norm(x.float(), (dim,), eps=1e-6))
    ref = torch.empty_like(ln)
    r0 = 0
    for i, r1 in enumerate(ends):
        t = E.bf(1 + sc[i].float())
        ref[r0:r1] = E.bf(E.bf(ln[r0:r1] * t) + sh[i].float())
        r0 = r1
    torch.testing.assert_close(out.float(), ref, rtol=2 ** -7, atol=2e-2)
    assert (out.float() == ref).float().mean().item() > 0.99


# ------------------------------------------------------------------------------------ per-module ranks end to end
RANKS = {"attn.to_q": 32, "attn.to_k": 64, "attn.to_v": 128, "proj_mlp": 96}


def test_per_module_ranks_match_the_oracle():
    """peft rank_pattern: to_q / to_k / to_v / proj_mlp with ranks 32 / 64 / 128 / 96 (others 48) and one alpha, so
    every module has its own alpha / r and the stacked q|k|v launches carry three different section scales.  Entry B
    with latent_lora and a 128x128 condition: the 256 image rows are fused, the 64 condition rows unfused."""
    from oracle import cases as C
    from oracle import flux_oracle as fo
    from reflectionflow_b200.transformer import B200FluxTransformer2DModel, tranformer_forward

    class PerModuleLora(fo.LoraSet):
        """peft's per-module scaling = alpha / r, r from that module's factors"""

        def __init__(self, weights, alpha):
            super().__init__(weights, 1.0)
            self.alpha = alpha

        def linear(self, name, lin, x, lora_on):
            y = lin(x)
            if name in self.weights:
                A, B = self.weights[name]
                s = self.alpha / A.shape[0] if lora_on else 0.0
                y = y + F.linear(F.linear(x, A.to(x.dtype)), B.to(x.dtype)) * s
            return y

    case = C.Case("fwdB_ll_ranks", cond_size=128, lora_rank=128, seed=81, model_config={"latent_lora": True})
    alpha = 64.0
    model, full = C.build_model(case)
    lora = {}
    for k, (a, b) in full.items():
        r = next((v for t, v in RANKS.items() if k.endswith(t)), 48)
        lora[k] = (a[:r].contiguous(), b[:, :r].contiguous())
    assert {32, 64, 128} <= {a.shape[0] for a, _ in lora.values()}
    x = C.build_inputs(case)
    mc = C.oracle_model_config(case)

    def oracle(m, ls, xx, **kw):
        with torch.no_grad():
            return fo.transformer_forward(m, xx["latents"], xx["prompt_embeds"], xx["pooled"], xx["timestep"],
                                          xx["img_ids"], xx["txt_ids"], xx["guidance"], xx["cond_latents"],
                                          xx["cond_ids"], mc, ls, **kw).float()
    ref = oracle(model, PerModuleLora(lora, alpha), x)
    single = oracle(model, fo.LoraSet(lora, alpha / case.lora_rank), x)
    m32 = model.float()
    l32 = {k: (a.float(), b.float()) for k, (a, b) in lora.items()}
    x32 = {k: (None if v is None else (v if k in ("timestep", "guidance") else v.float())) for k, v in x.items()}
    true32 = oracle(m32, PerModuleLora(l32, alpha), x32, scalar_dtype=torch.bfloat16)

    model, _ = C.build_model(case)
    m = B200FluxTransformer2DModel(case.config(), lora_rank=case.lora_rank)
    try:
        m.load_state_dict(model.state_dict())
        m.load_lora(lora, alpha=alpha)
        out = tranformer_forward(m, x["cond_latents"], x["cond_ids"], None, case.model_config, 0,
                                 hidden_states=x["latents"], encoder_hidden_states=x["prompt_embeds"],
                                 pooled_projections=x["pooled"], timestep=x["timestep"], img_ids=x["img_ids"],
                                 txt_ids=x["txt_ids"], guidance=x["guidance"], return_dict=False)[0]
        torch.cuda.synchronize()
        ours = out.cpu().float()
    finally:
        m.close()
    e_ours, e_ref, d = (ours - true32).abs(), (ref - true32).abs(), (ours - ref).abs()
    d_single = (ours - single).abs().mean()
    print(f"[per-module ranks] |ours-fp32| mean {e_ours.mean():.4g} max {e_ours.max():.4g} ; |ref-fp32| mean "
          f"{e_ref.mean():.4g} max {e_ref.max():.4g} ; |ours-ref| {d.mean():.4g} ; |ours-single scale| {d_single:.4g}")
    assert torch.isfinite(ours).all()
    assert e_ours.mean() <= 1.25 * e_ref.mean() + 1e-3
    assert e_ours.max() <= 2.0 * e_ref.max() + 1e-2
    assert d.mean() <= 2.0 * e_ref.mean() + 1e-3
    assert d.mean() < 0.25 * d_single
