"""References of the two attention kernels at their rounding points, the fixtures and bars the operator tests share, and
the ctypes binding of the text-attention test hook (csrc/rf_api.cu: rf_dbg_text_attention).

DiT attention (csrc/attn_sm90.cu) is an online softmax in log2 units.  `dit_attention` restates its order in float64
(or in fp32, to show the bars are reachable by fp32 arithmetic): the keys of each batch element are walked in 128-key
tiles, in order; per tile the running max m_t = max(m_{t-1}, max_j x_j) with x = s c + b log2(e), c = fp32(log2 e) *
fp32(1 / sqrt 128) as the kernel forms it; P = bf16(2^(x - m_t)) (rounded through fp32, as the kernel packs its fp32
P); l and O are rescaled by 2^(m_{t-1} - m_t), l adds the unrounded values and O adds P V; the output is bf16(O / l).
A row whose keys so far are all masked exponentiates against 0, so -inf - -inf never happens.  The mask comes from the
semantic definition only (`dit_mask`: block.py:106-122 element by element, keys >= n_tok dropped), never from the
kernel's cross / split / skip tile logic.

Text attention (csrc/text_attn_sm90.cu) keeps the rounding points of transformers' eager attention in bf16:
bf16(q k^T) [-> bf16(. * scale)] [-> bf16(. + bias[h, i, j])], mask (causal j <= i, keys < S), bf16(softmax_fp32),
bf16(P V) with P V in float64.  q and k come from the dyadic grids of tests/_exact.py, so q k^T is exact in fp32 and the
first rounding point is deterministic.

`mut` names one deliberate change (MUTATIONS); tests/test_attention_reference_host.py shows that each one fails the
bars of tests/test_gpu_attention.py on at least one of its fixtures."""
import math
import zlib
from ctypes import c_float, c_int, c_void_p

import torch

from tests import _exact as E

LOG2E = 1.4426950408889634
# the kernel's scale_log2: kLog2e * (1 / sqrt(128)), one fp32 multiply
C_LOG2 = (torch.tensor(LOG2E, dtype=torch.float32) * torch.tensor(0.08838834764831845, dtype=torch.float32)).item()
QSCALES = (0.0, 0.25, 1.0, 3.0)  # per query row i: QSCALES[i % 4] (row class i % 4); rows of class 0 are uniform

MUTATIONS = {
    # DiT attention
    "P_unrounded": "P used in P V without its bf16 rounding",
    "tail_unmasked": "keys past n_tok in the last partial tile not masked (score 0, V zero-filled)",
    "split_whole_tile": "the tile that holds the split masked / biased as a whole by its first row / key",
    "bias_unscaled": "cond_bias added to the raw score (the sqrt(128) factor lost)",
    "bias_one_way": "cond_bias / mask only on main queries x condition keys",
    "drop_kv_tile": "the last kv tile of every batch element skipped",
    # text attention
    "scores_unrounded": "q k^T not rounded to bf16",
    "bias_before_round": "bias added to q k^T before its bf16 rounding",
    "causal_off_by_one": "causal mask j <= i + 1",
    "bias_transposed": "bias read as bias[h, j, i]",
    "P_before_norm": "P rounded before the normalisation: bf16(bf16(e) V / sum)",
    "ragged_unmasked": "keys >= S of a batch element not masked (the next element's rows are read)",
}
DIT_MUTATIONS = ("P_unrounded", "tail_unmasked", "split_whole_tile", "bias_unscaled", "bias_one_way", "drop_kv_tile")
TEXT_MUTATIONS = ("scores_unrounded", "bias_before_round", "causal_off_by_one", "bias_transposed", "P_before_norm",
                  "ragged_unmasked")


def bf(x):
    """a bf16 rounding point (through fp32) of a float tensor, in its own dtype"""
    return x.float().to(torch.bfloat16).to(x.dtype)


def cond_bias(c):
    """log(c) rounded to bf16, as rf_dit_prepare builds it (the reference's mask is in the query dtype)"""
    return torch.tensor(math.log(c)).to(torch.bfloat16).item() if c > 0 else float("-inf")


# ------------------------------------------------------------------------------------ DiT attention
# name: (n_tok, heads, batch, n_main, cond_mode, c); cond_bias = cond_bias(c) for cond_mode 1
DIT_FIXTURES = {
    "n4608": (4608, 24, 1, None, 0, None),
    "n5632_m0": (5632, 24, 1, None, 0, None),
    "n5632_m1": (5632, 24, 1, 4608, 1, 2.0),
    "n5632_m2": (5632, 24, 1, 4608, 2, None),
    "n4544": (4544, 24, 1, None, 0, None),
    "n5120_m1": (5120, 24, 1, 4544, 1, 1.5),
    "n5120_m2": (5120, 24, 1, 4544, 2, None),
    "n5568_m1": (5568, 24, 1, 4544, 1, 2.0),
    "n5568_m2": (5568, 24, 1, 4544, 2, None),
    **{f"n{n}": (n, 2, 1, None, 0, None) for n in (1, 63, 128, 129, 255, 300)},
    **{f"n{n}_s{s}_m{m}": (n, 3 if n == 300 else 1, 1, s, m, (1.5, 2.0, 0.5, 1e-3)[i % 4] if m == 1 else None)
       for n in (300, 384) for i, s in enumerate((1, 77, 127, 128, 129)) for m in (1, 2)},
    "n300_s290_m1": (300, 2, 1, 290, 1, 0.5),
    "n300_s290_m2": (300, 2, 1, 290, 2, None),
    "n320_s256_m1": (320, 2, 1, 256, 1, 1e-3),
    "n320_s256_m2": (320, 2, 1, 256, 2, None),
    **{f"b3_n256_m{m}": (256, 2, 3, 200, m, 2.0 if m == 1 else None) for m in (0, 1, 2)},
    **{f"b3_n384_m{m}": (384, 2, 3, 256, m, 0.5 if m == 1 else None) for m in (0, 1, 2)},
}


def seed_of(name):
    return zlib.crc32(name.encode()) & 0x7FFFFFFF


def dit_fixture(name, device="cpu"):
    """-> (q, k, v, n_tok, heads, batch, n_main, mode, bias) of a DIT_FIXTURES entry"""
    n, heads, batch, n_main, mode, c = DIT_FIXTURES[name]
    q, k, v = split_qkv(dit_operands(n, heads, batch, seed_of(name), device), heads)
    return q, k, v, n, heads, batch, n_main, mode, cond_bias(c) if mode == 1 else 0.0


def probe_rows(n_tok, n_main=None):
    """rows 0..63, the query tile that holds the split and the last query tile (at most 256 rows)"""
    tiles = {(n_tok - 1) // 128}
    if n_main is not None:
        tiles.add(n_main // 128 if n_main < n_tok else (n_main - 1) // 128)
    rows = set(range(min(64, n_tok)))
    for t in tiles:
        rows |= set(range(t * 128, min((t + 1) * 128, n_tok)))
    return torch.tensor(sorted(rows))


def dit_operands(n_tok, heads, batch, seed, device="cpu"):
    """qkv [batch n_tok, 3 heads 128] bf16: query row i scaled by QSCALES[i % 4]; keys [5n/8, 6n/8) of every batch
    element scaled by 3, so the running max of the sharp rows moves late and the rescale of O and l matters"""
    inner = heads * 128
    g = torch.Generator(device="cpu").manual_seed(seed)
    qkv = torch.randn(batch, n_tok, 3 * inner, generator=g)
    qkv[:, :, :inner] *= torch.tensor(QSCALES)[torch.arange(n_tok) % 4][None, :, None]
    qkv[:, (5 * n_tok + 7) // 8:(6 * n_tok + 7) // 8, inner:2 * inner] *= 3.0
    return qkv.reshape(batch * n_tok, 3 * inner).to(torch.bfloat16).to(device)


def split_qkv(qkv, heads):
    inner = heads * 128
    return qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:]


def dit_mask(n_tok, n_main, mode, bias, mut=(), rows=None, device="cpu"):
    """the additive mask [rows, n_tok] in natural-log units, element by element (block.py:106-122): 0, or cond_bias
    (cond_mode 1) / -inf (cond_mode 2) between the tokens [0, n_main) and [n_main, n_tok)"""
    rows = torch.arange(n_tok, device=device) if rows is None else rows.to(device)
    m = torch.zeros(rows.numel(), n_tok, dtype=torch.float64, device=device)
    if mode == 0:
        return m
    keys = torch.arange(n_tok, device=device)
    if "split_whole_tile" in mut:
        rows, keys = rows // 128 * 128, keys // 128 * 128
    qc, kc = rows >= n_main, keys >= n_main
    cross = qc[:, None] != kc[None, :]
    if "bias_one_way" in mut:
        cross &= ~qc[:, None]
    m[cross] = float("-inf") if mode == 2 else bias
    return m


def dit_attention(q, k, v, heads, n_tok, batch=1, n_main=None, mode=0, bias=0.0, mut=(), dtype=torch.float64,
                  rows=None):
    """the kernel's order (module docstring) -> (out, A): out [batch len(rows), heads 128] holds bf16 values (dtype),
    A = sum_j p_j |v_j| with p the plain softmax, the magnitude the bars scale with.  `rows`: the query rows of each
    batch element to compute (default all)."""
    dev = q.device
    rows = torch.arange(n_tok, device=dev) if rows is None else rows.to(dev)
    R = rows.numel()
    T = (n_tok + 127) // 128
    c = torch.tensor(C_LOG2, dtype=dtype, device=dev)
    mask = dit_mask(n_tok, n_main, mode, bias, mut, rows, dev).to(dtype)
    madd = mask * (c if "bias_unscaled" in mut else LOG2E)
    out = torch.zeros(batch * R, heads * 128, dtype=dtype, device=dev)
    A = torch.zeros_like(out)
    for b in range(batch):
        for h in range(heads):
            cols = slice(h * 128, (h + 1) * 128)
            Q = q[b * n_tok + rows, cols].to(dtype)
            K = k[b * n_tok:(b + 1) * n_tok, cols].to(dtype)
            V = v[b * n_tok:(b + 1) * n_tok, cols].to(dtype)
            X = (Q @ K.t()) * c + madd
            # the plain softmax: the bars' magnitude
            p = torch.softmax(X * math.log(2.0), dim=1)
            A[b * R:(b + 1) * R, cols] = p @ V.abs()
            pad = T * 128 - n_tok
            X = torch.nn.functional.pad(X, (0, pad), value=0.0 if "tail_unmasked" in mut else float("-inf"))
            V = torch.nn.functional.pad(V, (0, 0, 0, pad))
            m = torch.full((R,), float("-inf"), dtype=dtype, device=dev)
            l = torch.zeros(R, dtype=dtype, device=dev)
            O = torch.zeros(R, 128, dtype=dtype, device=dev)
            for t in range(T):
                if "drop_kv_tile" in mut and t == T - 1:
                    continue
                xt = X[:, t * 128:(t + 1) * 128]
                m_new = torch.maximum(m, xt.max(dim=1).values)
                m_use = torch.where(m_new == float("-inf"), torch.zeros_like(m_new), m_new)
                alpha = torch.exp2(m - m_use)
                e = torch.exp2(xt - m_use[:, None])
                P = e if "P_unrounded" in mut else bf(e)
                l = l * alpha + e.sum(dim=1)
                O = O * alpha[:, None] + P @ V[t * 128:(t + 1) * 128]
                m = m_new
            o = torch.where(l[:, None] > 0, O / l.clamp_min(torch.finfo(dtype).tiny)[:, None], torch.zeros_like(O))
            out[b * R:(b + 1) * R, cols] = bf(o)
    return out, A


def dit_plain(q, k, v, heads, n_tok, batch=1, n_main=None, mode=0, bias=0.0):
    """the plain float64 softmax attention (no rounding point) over the same mask, [batch n_tok, heads 128]"""
    out = torch.zeros(batch * n_tok, heads * 128, dtype=torch.float64, device=q.device)
    mask = dit_mask(n_tok, n_main, mode, bias, device=q.device)
    for b in range(batch):
        r = slice(b * n_tok, (b + 1) * n_tok)
        for h in range(heads):
            cols = slice(h * 128, (h + 1) * 128)
            s = q[r, cols].double() @ k[r, cols].double().t() / math.sqrt(128.0) + mask
            out[r, cols] = torch.softmax(s, dim=1) @ v[r, cols].double()
    return out


def ulp_bf16(ref):
    """the bf16 spacing at |ref| (2^(e - 7) for |ref| in [2^e, 2^(e + 1))); 0 maps to the least subnormal"""
    a = ref.double().abs()
    e = torch.floor(torch.log2(torch.where(a > 0, a, torch.ones_like(a))))
    return torch.where(a > 0, torch.exp2(e - 7), torch.full_like(a, 2.0 ** -133))


def within_bar(out, ref, A):
    """per element: |out - ref| <= 1 ulp_bf16(ref) + 2^-7 A, A = sum_j p_j |v_j|.  The kernel and the reference each
    round every P to bf16; where an fp32 exp lands on the other side of a rounding midpoint the two P differ by one
    bf16 ulp, up to 2^-7 P (for P just above a power of two), so their P V differ by at most 2^-7 A, and the two output
    roundings add at most 1 ulp.  2^-8 A is not enough: the fp32 restatement itself exceeds it on sharp rows whose
    second-largest weight lies in [0.5, 1)."""
    d = (out.double() - ref.double()).abs()
    return d <= ulp_bf16(ref) + 2.0 ** -7 * A.double()


DIT_IDENTICAL = 0.99  # the bit-identical fraction every row class of every fixture must reach


def dit_check(out, ref, A, rows, heads, batch=1):
    """-> (all elements within the bar, {row class: bit-identical fraction}) for outputs [batch len(rows), heads 128]
    of the query rows `rows` of each batch element"""
    ok = within_bar(out, ref, A) & torch.isfinite(out)
    same = (out.double() == ref.double()).view(batch, rows.numel(), heads * 128)
    cls = (rows.to(out.device) % 4)
    fr = {k: same[:, cls == k].double().mean().item() for k in range(4) if bool((cls == k).any())}
    return bool(ok.all()), fr


def dit_passes(out, ref, A, rows, heads, batch=1):
    ok, fr = dit_check(out, ref, A, rows, heads, batch)
    return ok and min(fr.values()) >= DIT_IDENTICAL


# ------------------------------------------------------------------------------------ text attention
# name: (B, S, heads, kind, bias_offset); kind "t5": random asymmetric bias, no scale; "clip": scale 1/8, causal
TEXT_FIXTURES = {
    **{f"t5_S{S}_h{h}_B{B}": (B, S, h, "t5", 0)
       for S in (1, 2, 63, 64, 65, 77, 127, 128, 129, 255, 256, 300, 511, 512)
       for h, B in ((1, 3), (4, 1), (64, 1) if S in (77, 512) else (4, 3))},
    "t5_S256_h4_B1_off2": (1, 256, 4, "t5", 2),
    "t5_S512_h4_B3_off2": (3, 512, 4, "t5", 2),
    **{f"clip_S{S}_h{h}_B{B}": (B, S, h, "clip", 0) for S in (77, 300) for h, B in ((4, 3), (12, 1))},
}


def text_operands(B, S, heads, kind, offset, seed, device="cpu"):
    """q = k/8 (|k| <= 16), k = k/16 (|k| <= 8): q k^T is exact in fp32 (products on a 2^-7 grid, at most 64 of
    magnitude <= 1); v random; the T5 bias [heads, S, S] is an asymmetric random bf16 tensor, viewed `offset`
    elements into its storage"""
    inner = heads * 64
    q = E.dyadic((B * S, inner), 3, 16, seed)
    kk = E.dyadic((B * S, inner), 4, 8, seed + 1)
    v = E.randn((B * S, inner), seed + 2)
    qkv = torch.cat([q, kk, v], dim=1).to(device)
    bias = None
    if kind == "t5":
        g = torch.Generator(device="cpu").manual_seed(seed + 3)
        raw = torch.randn(heads * S * S + offset, generator=g) * 1.5 + torch.linspace(-1.0, 1.0, heads * S * S + offset)
        bias = raw.to(torch.bfloat16).to(device)[offset:].view(heads, S, S)
    return qkv, bias


def _text_keys(t, b, S, cols, mut):
    """the keys / values batch element b attends to: its S rows, or (ragged_unmasked) the whole 128-row blocks the
    kernel loads, which run into the next element's rows (zero past the end)"""
    nk = (S + 127) // 128 * 128 if "ragged_unmasked" in mut else S
    out = torch.zeros(nk, 64, dtype=torch.float64, device=t.device)
    src = t[b * S:b * S + nk, cols].double()
    out[:src.shape[0]] = src
    return out


def text_scores(q, k, b, h, S, bias=None, scale=1.0, use_scale=False, causal=False, mut=()):
    """the masked bf16 scores [S, keys] of batch element b, head h (fp32 holding bf16 values, -inf where masked)"""
    cols = slice(h * 64, (h + 1) * 64)
    s = q[b * S:(b + 1) * S, cols].double() @ _text_keys(k, b, S, cols, mut).t()
    nk = s.shape[1]
    assert torch.equal(s.float().double(), s), "q k^T not exact in fp32"
    s = s.float()
    bb = None
    if bias is not None:
        bb = torch.zeros(S, nk, dtype=torch.float32, device=s.device)
        bh = bias[h].float()
        bb[:, :S] = bh.t() if "bias_transposed" in mut else bh
    if "bias_before_round" in mut and bb is not None:
        y = bf(s + bb)
    else:
        y = s if "scores_unrounded" in mut else bf(s)
        if use_scale:
            y = bf(y * E.f32(scale).to(s.device))
        if bb is not None:
            y = bf(y + bb)
    i = torch.arange(S, device=s.device)[:, None]
    j = torch.arange(nk, device=s.device)[None, :]
    masked = (j >= S) if "ragged_unmasked" not in mut else torch.zeros_like(j, dtype=torch.bool)
    if causal:
        masked = masked | (j > i + (1 if "causal_off_by_one" in mut else 0))
    return y.masked_fill(masked, float("-inf"))


def text_attention(q, k, v, B, S, heads, bias=None, scale=1.0, use_scale=False, causal=False, mut=()):
    """eager attention at its bf16 rounding points -> (out, A): out [B S, heads 64] fp32 holding bf16 values, A = P |V|,
    the magnitude the bars scale with"""
    out = torch.zeros(B * S, heads * 64, dtype=torch.float32, device=q.device)
    A = torch.zeros(B * S, heads * 64, dtype=torch.float64, device=q.device)
    for b in range(B):
        for h in range(heads):
            cols = slice(h * 64, (h + 1) * 64)
            y = text_scores(q, k, b, h, S, bias, scale, use_scale, causal, mut)
            V = _text_keys(v, b, S, cols, mut)
            if "P_before_norm" in mut:
                e = torch.exp(y - y.max(dim=1, keepdim=True).values)
                P = bf(e).double() / e.sum(dim=1, keepdim=True).double()
            else:
                P = bf(torch.softmax(y, dim=1)).double()
            out[b * S:(b + 1) * S, cols] = bf((P @ V).float())
            A[b * S:(b + 1) * S, cols] = P @ V.abs()
    return out, A


TEXT_IDENTICAL = 0.999  # the bit-identical fraction every text fixture must reach


def text_passes(out, ref, A):
    """within_bar everywhere (with A = P |V|: the kernel's expf and its e * (1 / sum) are not torch's softmax bit for
    bit, so a few P land one bf16 ulp away) and TEXT_IDENTICAL bit-identical"""
    ok = torch.isfinite(out).all() and bool(within_bar(out, ref, A).all())
    return bool(ok) and (out == ref).double().mean().item() >= TEXT_IDENTICAL


def text_args(kind):
    """(scale, use_scale, causal) of a fixture kind"""
    return (1.0, 0, 0) if kind == "t5" else (0.125, 1, 1)


# ------------------------------------------------------------------------------------ test-hook binding
def declare(lib):
    vp, ci = c_void_p, c_int
    lib.rf_dbg_text_attention.restype = ci
    lib.rf_dbg_text_attention.argtypes = [vp, vp, vp, ci, vp, ci, ci, ci, ci, vp, c_float, ci, ci, vp]
    return lib
