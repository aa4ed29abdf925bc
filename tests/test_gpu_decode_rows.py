"""The decode step at 65-256 rows per session, and the kernels that consume its split-K partials, against float64 references.

A session pads its B decode rows to Bp = round_up(B, 16), and every swap-AB decoder GEMM runs with bn = Bp rounded up to a power of two:
Bp = 80..128 runs 128-column tiles and Bp = 144..256 runs 256-column tiles, up to 96 of whose columns are TMA zero-fill that the
GEMM_OUT_PARTIAL_T epilogue must drop.  The benchmarked configurations run 128 (large-v3-turbo greedy, 1024 windows on 8 GPUs) and 160
(large-v3 beam 5, 256 windows on 8 GPUs) rows per GPU.  This file checks, on the same 16-bit inputs:

  * the raw split-K partials [splits][partial_cols][N] of the GEMM, slab by slab, at every production (N, K) of d = 384 / 768 / 1280,
    inside a NaN-guarded buffer (nothing may be written outside it), in both the layer form and the logits form (partial_cols = B < Bp);
  * the partial consumers - reduce + bias + residual + LayerNorm, reduce + bias + GELU, the q/k/v reduction of self-attention (with beam
    cache ancestry) and the q reduction of cross-attention (single-query, beam and FP8-cache kernels) - with garbage in partial rows >= B;
  * end to end at large-v3 width: 130 greedy windows in one session (Bp = 144) against the same-policy oracle twin and against each window
    decoded alone, and 32 windows x 5 beams (160 rows) against each window alone and against the beam oracle.

Tolerances are bounds derived from the arithmetic (f32 unit roundoff u = 2^-24 times the number of roundings on the path times the
magnitudes involved, plus one ulp of the 16-bit storage type where a result is stored in it); each case prints the measured worst error
as a fraction of its bound."""
import ctypes as C
import dataclasses
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from whisperkit_b200 import _lib  # noqa: E402
from oracle import beam_ref as BR  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from oracle import model_ref as M  # noqa: E402
from tests import fp8_ref  # noqa: E402
from tests.test_gpu_beam import _predictor  # noqa: E402
from tests.test_gpu_large import LV3, TOL_TWIN, rel_err  # noqa: E402

TD = {"bf16": (torch.bfloat16, _lib.WK_DTYPE_BF16), "f16": (torch.float16, _lib.WK_DTYPE_F16)}
U = 2.0 ** -24                      # f32 unit roundoff: one IEEE round-to-nearest step moves a value by at most U times its magnitude
SIG_BITS = {"bf16": 8, "f16": 11}   # significand bits of the storage types (implicit bit included)
B_LIST = [1, 17, 64, 130, 160]      # Bp = 16, 32, 64, 144, 160
KV_MAX = 224
GUARD = 4096                        # NaN guard elements on either side of a buffer the kernels write


@pytest.fixture(scope="module")
def toy():
    m = wk.Model("toy", max_batch=4)
    m.init_random(seed=3)
    yield m
    m.close()


def p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def round_up(a, b):
    return (a + b - 1) // b * b


def tile_n(bn):
    """wgmma_tile_n (gemm_wgmma.cu): the wgmma tile width a GEMM with bn columns runs with."""
    t = 16
    while t < bn:
        t <<= 1
    return t


def choose_splits(tiles, total_kb, num_sms):
    """engine.cu choose_splits: the deepest split-K (<= 20) dividing the k-blocks that keeps tiles * splits within one wave."""
    best = 1
    for s in range(1, min(total_kb, 20) + 1):
        if total_kb % s == 0 and tiles * s <= num_sms:
            best = s
    return best


def deepest_split(total_kb):
    return max(s for s in range(1, 21) if total_kb % s == 0)


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def ulp16(v, dt):
    """Spacing of the 16-bit storage type at |v| (f16: its subnormal spacing 2^-24 below 2^-14)."""
    e = torch.floor(torch.log2(v.abs().double().clamp_min(1e-300)))
    if dt == "f16":
        e = e.clamp_min(-14)
    return torch.exp2(e - (SIG_BITS[dt] - 1))


def check(name, err, bound):
    """err, bound: tensors of the same shape.  NaN in err fails."""
    ratio = (err / bound).max().item() if err.numel() else 0.0
    bad = int((~(err <= bound)).sum().item())
    print(f"[{name}] worst error {err.max().item():.3e}, {ratio:.3f} of its bound")
    assert bad == 0, f"{name}: {bad} elements outside the bound (worst ratio {ratio})"


def guarded(n, pre=GUARD, post=GUARD, dtype=torch.float32):
    buf = torch.full((pre + n + post,), float("nan"), device="cuda", dtype=dtype)
    return buf, buf[pre:pre + n]


def guards_untouched(buf, pre, n):
    return bool(torch.isnan(buf[:pre]).all().item()) and bool(torch.isnan(buf[pre + n:]).all().item())


# ================================================================================== 1. swap-AB split-K GEMM partials
GEMM_SHAPES = [(n, k) for d in (384, 768, 1280) for (n, k) in ((3 * d, d), (d, d), (4 * d, d), (d, 4 * d), (51866, d))]
GEMM_ROWS = [16, 48, 64, 80, 112, 128, 144, 160, 208, 256]


def run_partial(toy, w, x, N, rows, pcols, K, wdt, splits):
    """Raw partials of one GEMM into a NaN-guarded buffer.  The trailing guard covers every column up to the wgmma tile width, so a store
    of the zero-filled columns lands in it (and fails the test) instead of outside the allocation."""
    n = splits * pcols * N
    post = (tile_n(rows) - pcols) * N + GUARD
    buf, part = guarded(n, GUARD, post)
    torch.cuda.synchronize()
    _lib.check(toy.lib.wk_test_gemm_partial(toy.handle, p(w), p(x), p(part), N, rows, pcols, K, wdt, splits))
    torch.cuda.synchronize()
    assert guards_untouched(buf, GUARD, n), f"the GEMM wrote outside its partial buffer (rows {rows}, partial_cols {pcols}, splits {splits})"
    return part.view(splits, pcols, N)


def check_slabs(name, part, x, w, splits, pcols):
    """Slab s must be x[:pcols] . w^T over k-blocks [s K / splits, (s + 1) K / splits) alone.  Bound: the 16-bit products are exact in f32
    (8 x 8 or 11 x 11 significand bits), and the f32 accumulation of a slab rounds at most once per term, each time by at most 2 U (the
    tensor core may truncate rather than round) times the running sum, itself at most sum |x||w| over the slice:
        |err| <= 2 U * (K / splits) * sum_k |x_k w_k|."""
    K = x.shape[1]
    ks = K // splits
    worst = 0.0
    for s in range(splits):
        xs, ws = x[:pcols, s * ks:(s + 1) * ks].double(), w[:, s * ks:(s + 1) * ks].double()
        ref = xs @ ws.t()
        bound = 2 * U * ks * (xs.abs() @ ws.abs().t())
        err = (part[s].double() - ref).abs()
        bad = int((~(err <= bound)).sum().item())
        assert bad == 0, f"{name}: split {s}: {bad} elements outside the bound (max err {err.max().item():.3e})"
        worst = max(worst, (err / bound).max().item())
    return worst


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("N,K", GEMM_SHAPES)
def test_gemm_partial_slabs_at_every_row_count(toy, dt, N, K):
    """Layer form (partial_cols = Bp): every production (N, K) of d = 384 / 768 / 1280 at Bp = 16 .. 256, with the split-K depth the decode
    step picks on this device, no split, and the deepest split (<= 20) that divides the k-blocks."""
    tdt, wdt = TD[dt]
    g = torch.Generator(device="cuda").manual_seed(N * 7 + K)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(tdt)
    xall = torch.randn(256, K, device="cuda", generator=g).to(tdt)
    kb = K // 64
    split_set = sorted({choose_splits((N + 127) // 128, kb, num_sms()), 1, deepest_split(kb)})
    worst = 0.0
    for rows in GEMM_ROWS:
        x = xall[:rows].contiguous()
        for sp in split_set:
            part = run_partial(toy, w, x, N, rows, rows, K, wdt, sp)
            worst = max(worst, check_slabs(f"{N}x{K} rows {rows} splits {sp}", part, x, w, sp, rows))
    print(f"[gemm partial {dt} {N}x{K}, splits {split_set}] worst error {worst:.3f} of its bound")


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("K", [384, 768, 1280])
@pytest.mark.parametrize("B", [17, 65, 129, 130, 250])
def test_gemm_partial_logits_form_drops_padded_columns(toy, dt, K, B):
    """Logits form: the activations have Bp = round_up(B, 16) rows but only columns < B are stored (partial_cols = B, splits 1).  Rows B..Bp-1
    of x hold live values here, so any of their columns that were stored would land in the trailing guard."""
    tdt, wdt = TD[dt]
    N, rows = 51866, round_up(B, 16)
    g = torch.Generator(device="cuda").manual_seed(B * 13 + K)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(tdt)
    x = torch.randn(rows, K, device="cuda", generator=g).to(tdt)
    part = run_partial(toy, w, x, N, rows, B, K, wdt, 1)
    worst = check_slabs(f"logits {K} B {B}", part, x, w, 1, B)
    print(f"[gemm logits form {dt} K {K} B {B} Bp {rows}] worst error {worst:.3f} of its bound")


# ================================================================================== 2. split-K consumers
def make_partials(g, splits, Bp, B, n, scale):
    """[splits][Bp][n] f32; rows B..Bp-1 are NaN (whatever the GEMM left in the padded columns must never reach an output)."""
    part = torch.randn(splits, Bp, n, device="cuda", generator=g) * scale
    part[:, B:] = float("nan")
    return part


def emulate_f32_sum(start, part, B):
    """start + part[0] + part[1] + ... in f32, in the kernels' order (bit-exact: IEEE adds)."""
    acc = start
    for s in range(part.shape[0]):
        acc = acc + part[s, :B]
    return acc


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("d", [384, 1280])
@pytest.mark.parametrize("B", B_LIST)
@pytest.mark.parametrize("with_bias", [True, False])
def test_reduce_residual_layernorm(toy, dt, d, B, with_bias):
    """decoder_reduce_resid_ln at splits 1..20: x += bias + sum_s partial[s] (f32, in place), xn = LN(x) (16-bit).

    x: the kernel adds bias and then the splits in order, splits + 1 roundings each bounded by U times the running sum's magnitude:
        |err x| <= (splits + 1) U (|x0| + |bias| + sum_s |p_s|).
    xn, against float64 LN of the GPU's own x: the mean and variance reductions are trees of at most 8 sequential adds in a thread, 5
    warp-shuffle levels and 5 levels over the warps (+ the division): D = 20 roundings, so the mean is off by at most D U mean|x| <=
    D U max|x| and the variance / rstd relatively by about D U.  Hence
        |err xn| <= ulp16(xn) + D U (|gamma| rstd max|x| + |xn| + |beta|).
    Row B // 2 sits at x = 1000 + N(0, 1): there max|x| / std = 1000, which a one-pass variance (E[x^2] - mean^2) cannot survive."""
    tdt, wdt = TD[dt]
    Bp = round_up(B, 16)
    g = torch.Generator(device="cuda").manual_seed(B * 31 + d + with_bias)
    gamma = 1.0 + 0.1 * torch.randn(d, device="cuda", generator=g)
    beta = 0.1 * torch.randn(d, device="cuda", generator=g)
    bias = 0.1 * torch.randn(d, device="cuda", generator=g) if with_bias else None
    worst_x, worst_n = 0.0, 0.0
    for splits in range(1, 21):
        part = make_partials(g, splits, Bp, B, d, 0.5)
        x0 = torch.randn(B, d, device="cuda", generator=g) * 2.0
        x0[B // 2] = 1000.0 + torch.randn(d, device="cuda", generator=g)
        xbuf = torch.full((Bp, d), 7.0, device="cuda")
        xbuf[:B] = x0
        out = torch.full((Bp, d), 7.0, device="cuda", dtype=tdt)
        torch.cuda.synchronize()
        _lib.check(toy.lib.wk_test_decoder_reduce(toy.handle, 0, p(part), splits, Bp, p(bias), p(gamma), p(beta), p(xbuf), p(out), B, d, wdt))
        torch.cuda.synchronize()
        pv = part[:, :B].double()
        bias64 = bias.double() if bias is not None else torch.zeros(d, device="cuda", dtype=torch.float64)
        ref_x = x0.double() + bias64 + pv.sum(0)
        mag = x0.double().abs() + bias64.abs() + pv.abs().sum(0)
        err_x = (xbuf[:B].double() - ref_x).abs()
        bound_x = (splits + 1) * U * mag
        assert int((~(err_x <= bound_x)).sum().item()) == 0, f"x: splits {splits}, max err {err_x.max().item():.3e}"
        worst_x = max(worst_x, (err_x / bound_x).max().item())
        xg = xbuf[:B].double()
        mean = xg.mean(1, keepdim=True)
        rstd = 1.0 / torch.sqrt(((xg - mean) ** 2).mean(1, keepdim=True) + 1e-5)
        ref = (xg - mean) * rstd * gamma.double() + beta.double()
        bound = ulp16(ref, dt) + 20 * U * (gamma.double().abs() * rstd * xg.abs().amax(1, keepdim=True) + ref.abs() + beta.double().abs())
        err = (out[:B].double() - ref).abs()
        assert int((~(err <= bound)).sum().item()) == 0, f"xn: splits {splits}, max err {err.max().item():.3e}"
        worst_n = max(worst_n, (err / bound).max().item())
        assert torch.all(xbuf[B:] == 7.0) and torch.all(out[B:].float() == 7.0), "rows past B were written"
    print(f"[reduce+LN {dt} d {d} B {B} bias {with_bias}] worst error over splits 1..20: x {worst_x:.3f}, xn {worst_n:.3f} of the bounds")


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("d", [384, 1280])
@pytest.mark.parametrize("B", B_LIST)
def test_reduce_bias_gelu(toy, dt, d, B):
    """decoder_reduce_bias_gelu at splits 1..20 (splits > 8 run the kernel's separate tail loop): out = gelu(bias + sum_s partial[s]),
    exact-erf GELU, 16-bit, n = 4 d.  Bound against float64:
        ulp16(out) + 1.13 (splits + 1) U (|bias| + sum_s |p_s|)      the f32 sum (GELU's slope is at most 1.13)
                   + 0.5 |a| (1.5e-7 + 16 U)                          erf by Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7) in f32."""
    tdt, wdt = TD[dt]
    n, Bp = 4 * d, round_up(B, 16)
    g = torch.Generator(device="cuda").manual_seed(B * 17 + d)
    bias = 0.5 * torch.randn(n, device="cuda", generator=g)
    worst = 0.0
    for splits in range(1, 21):
        part = make_partials(g, splits, Bp, B, n, 0.7)
        out = torch.full((Bp, n), 7.0, device="cuda", dtype=tdt)
        torch.cuda.synchronize()
        _lib.check(toy.lib.wk_test_decoder_reduce(toy.handle, 1, p(part), splits, Bp, p(bias), None, None, None, p(out), B, n, wdt))
        torch.cuda.synchronize()
        pv = part[:, :B].double()
        a = bias.double() + pv.sum(0)
        ref = 0.5 * a * (1.0 + torch.special.erf(a / math.sqrt(2.0)))
        bound = ulp16(ref, dt) + 1.13 * (splits + 1) * U * (bias.double().abs() + pv.abs().sum(0)) + 0.5 * a.abs() * (1.5e-7 + 16 * U)
        err = (out[:B].double() - ref).abs()
        assert int((~(err <= bound)).sum().item()) == 0, f"splits {splits}: max err {err.max().item():.3e}"
        worst = max(worst, (err / bound).max().item())
        assert torch.all(out[B:].float() == 7.0), "rows past B were written"
    print(f"[reduce+GELU {dt} d {d} B {B}] worst error over splits 1..20: {worst:.3f} of the bound")


def attention_bound(q, qmag, n_q_terms, Kx, Vx, valid, ref, dt, hilo=False):
    """Bound on |out - ref| of one-query attention computed in f32 (kernels of decoder_ops.cu / cross_attention_mq.cu), float64 ref.
    q [R,H,64] exact query, qmag the magnitude sum it was reduced from, n_q_terms the f32 adds that made it; Kx / Vx [R,H,T,64] the
    stored keys / values, valid [R,1,T] mask.  `st` is the bound of one accumulation step: U on the FMA pipe, 2 U on the tensor cores
    (hilo: the beam kernel), whose f32 accumulation may truncate instead of rounding.
      score error   ds_t <= 0.125 (n_q_terms + 64 st / U + 4) U sum_j qmag_j |k_tj|   (q reduction, 64-term dot, scales)
      (hilo: its hi + lo 16-bit split of the scaled query q / 8 keeps 16 significand bits, down to the f16 subnormal spacing 2^-25 of the
      lo half: + sum_j (2^-16 |q_j| / 8 + 2^-25) |k_tj|)
      softmax       p_t moves relatively by at most 2 max_t ds_t + (|s_t - max s| + 8) U (exp2 of a rounded argument, normalisation)
      output        sum_t p_t v_t over n terms: + (n st / U + 32) U max|v|  (accumulation and the fixed roundings around it)
      (hilo: the hi + lo split of p: + (2^-16 + n 2^-35) max|v|)
    plus one ulp of the 16-bit output."""
    st = 2 if hilo else 1
    scores_mag = torch.einsum("rhd,rhtd->rht", qmag, Kx.abs()) * 0.125
    ds = (n_q_terms + 64 * st + 4) * U * scores_mag
    if hilo:
        ds = ds + torch.einsum("rhd,rhtd->rht", 2.0 ** -16 * q.abs() * 0.125 + 2.0 ** -25, Kx.abs())
    s = torch.einsum("rhd,rhtd->rht", q, Kx) * 0.125
    s = s.masked_fill(~valid, float("-inf"))
    srange = (s.amax(-1) - s.masked_fill(~valid, float("inf")).amin(-1))
    ds_max = ds.masked_fill(~valid, 0.0).amax(-1)
    vmax = Vx.abs().masked_fill(~valid[..., None], 0.0).amax(dim=(-1, -2))
    n = valid.sum(-1).double()
    rel = 2 * ds_max + (srange + 8) * U + (n * st + 32) * U
    if hilo:
        rel = rel + 2.0 ** -16 + n * 2.0 ** -35
    return ulp16(ref, dt) + (vmax * rel)[..., None]


def attention_ref(q, Kx, Vx, valid):
    s = torch.einsum("rhd,rhtd->rht", q, Kx) * 0.125
    pr = torch.softmax(s.masked_fill(~valid, float("-inf")), dim=-1)
    return torch.einsum("rht,rhtd->rhd", pr, Vx)


def self_attn_cases():
    cases = []
    for B in B_LIST:
        cases.append((B, 0))
        beam = next((b for b in (5, 4) if B % b == 0 and B > b), 0)
        if beam:
            cases.append((B, beam))
    return cases


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("d", [384, 1280])
@pytest.mark.parametrize("B,beam", self_attn_cases())
def test_self_attention_splitk(toy, dt, d, B, beam):
    """decoder_self_attention_kernel as the step runs it: q|k|v reduced from split-K partials (rows >= B NaN) plus bq / bv, the new K/V row
    appended at pos[b] (positions 0 and 223 included), rows flagged done untouched.  beam > 0: rows come in windows of `beam`, all beams of a
    window at one position, and anc[b][t] sends position t of beam b to a random beam's cache row of the same window; the reference gathers
    through it, and the new row must still land in row b's own cache, rounded to the storage type (bit-exact against the f32 sum)."""
    tdt, wdt = TD[dt]
    H, Bp = d // 64, round_up(B, 16)
    dm = H * 64
    g = torch.Generator(device="cuda").manual_seed(B * 11 + d + beam)
    gc = torch.Generator().manual_seed(B * 11 + d + beam)
    kb = d // 64
    for splits in sorted({choose_splits((3 * d + 127) // 128, kb, num_sms()), deepest_split(kb)}):
        part = make_partials(g, splits, Bp, B, 3 * dm, 0.5)
        bq = 0.3 * torch.randn(dm, device="cuda", generator=g)
        bv = 0.3 * torch.randn(dm, device="cuda", generator=g)
        kc0 = torch.randn(B, H, KV_MAX, 64, device="cuda", generator=g).to(tdt)
        vc0 = torch.randn(B, H, KV_MAX, 64, device="cuda", generator=g).to(tdt)
        groups = B // beam if beam else B
        gpos = [0, KV_MAX - 1] + [int(v) for v in torch.randint(0, KV_MAX, (max(0, groups - 2),), generator=gc)]
        gpos = gpos[:groups]
        pos_l = [gpos[b // beam] if beam else gpos[b] for b in range(B)]
        pos = torch.tensor(pos_l, dtype=torch.int32, device="cuda")
        done = torch.zeros(B, dtype=torch.int32, device="cuda")
        if B > 2:
            dw = (groups - 1) if beam else B - 1          # the last window (all its beams) has ended
            done[dw * (beam or 1):(dw + 1) * (beam or 1)] = 1
        anc = None
        if beam:
            own = (torch.arange(B) // beam * beam)[:, None]
            anc = (own + torch.randint(0, beam, (B, KV_MAX), generator=gc)).to(torch.int32).cuda()
            assert (anc != torch.arange(B, device="cuda")[:, None].int()).float().mean() > 0.5
        kc, vc = kc0.clone(), vc0.clone()
        out = torch.full((B, dm), 7.0, device="cuda", dtype=tdt)
        torch.cuda.synchronize()
        _lib.check(toy.lib.wk_test_self_attention_splitk(toy.handle, p(part), splits, Bp, p(bq), p(bv), p(kc), p(vc), p(pos), p(done), p(anc),
                                                         p(out), B, H, wdt))
        torch.cuda.synchronize()
        live = done == 0
        rows = torch.arange(B, device="cuda")
        # the appended row: the f32 reduction (q from bq, k from 0, v from bv, then the splits in order) rounded to the storage type
        knew = emulate_f32_sum(torch.zeros(dm, device="cuda"), part[:, :, dm:2 * dm], B).reshape(B, H, 64).to(tdt)
        vnew = emulate_f32_sum(bv, part[:, :, 2 * dm:], B).reshape(B, H, 64).to(tdt)
        kexp, vexp = kc0.clone(), vc0.clone()
        lr, lp = rows[live], pos.long()[live]
        kexp[lr, :, lp] = knew[live]
        vexp[lr, :, lp] = vnew[live]
        assert torch.equal(kc, kexp) and torch.equal(vc, vexp), "cache: the new row is wrong, misplaced, or another row changed"
        assert torch.all(out[~live].float() == 7.0), "a done row was written"
        # reference: positions < pos read through anc from the ORIGINAL caches, position pos is the new row
        pv = part[:, :B].double()
        q = (bq.double() + pv[:, :, :dm].sum(0)).view(B, H, 64)
        qmag = (bq.double().abs() + pv[:, :, :dm].abs().sum(0)).view(B, H, 64)
        src = anc.long() if beam else rows[:, None].expand(B, KV_MAX)
        tt = torch.arange(KV_MAX, device="cuda")
        Kx = kc0.permute(0, 2, 1, 3)[src, tt[None, :]].permute(0, 2, 1, 3).double()    # [B, H, 224, 64]
        Vx = vc0.permute(0, 2, 1, 3)[src, tt[None, :]].permute(0, 2, 1, 3).double()
        Kx[rows, :, pos.long()] = knew.double()
        Vx[rows, :, pos.long()] = vnew.double()
        valid = (tt[None, :] <= pos.long()[:, None])[:, None, :]                      # [B, 1, 224]
        ref = attention_ref(q, Kx, Vx, valid)
        bound = attention_bound(q, qmag, splits + 1, Kx, Vx, valid, ref, dt)
        err = (out.view(B, H, 64).double() - ref).abs()
        check(f"self-attention {dt} d {d} B {B} beam {beam} splits {splits}", err[live], bound[live])


def cross_cases():
    cases = [(B, 1, False) for B in B_LIST] + [(17, 1, True)]
    cases += [(B, 5, fp8) for B in (130, 160) for fp8 in (False, True)]
    return cases


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("d", [384, 1280])
@pytest.mark.parametrize("B,kv_div,fp8", cross_cases())
def test_cross_attention_splitk(toy, dt, d, B, kv_div, fp8):
    """Decoder cross-attention over T = 1500 with q reduced from split-K partials (rows >= B NaN) plus bcq: the single-query kernel
    (kv_div = 1) and the beam kernel (kv_div = 5: 5 rows share one K/V block; B = 160 is 32 windows x 5 beams), 16-bit or FP8 cache (E4M3
    codes with one f32 scale per row, tests/fp8_ref.py layout).  The reference uses the stored K/V (dequantized for FP8) in float64."""
    tdt, wdt = TD[dt]
    H, Bp, T = d // 64, round_up(B, 16), 1500
    dm, W = H * 64, B // kv_div
    g = torch.Generator(device="cuda").manual_seed(B * 5 + d + kv_div + fp8)
    kb = d // 64
    splits = choose_splits((d + 127) // 128, kb, num_sms())
    splits = splits if splits > 1 else deepest_split(kb)
    part = make_partials(g, splits, Bp, B, dm, 0.4)
    bq = 0.3 * torch.randn(dm, device="cuda", generator=g)
    kf = torch.randn(W, H, T, 64, device="cuda", generator=g) * 0.7
    vf = torch.randn(W, H, T, 64, device="cuda", generator=g)
    if fp8:
        kcode, ksc = fp8_ref.quantize_rows(kf)
        vcode, vsc = fp8_ref.quantize_rows(vf)
        kcode, vcode, ksc, vsc = kcode.contiguous(), vcode.contiguous(), ksc.contiguous(), vsc.contiguous()
        kst, vst = kcode, vcode
        K64, V64 = fp8_ref.dequantize_rows(kcode, ksc).double(), fp8_ref.dequantize_rows(vcode, vsc).double()
    else:
        kst, vst = kf.to(tdt), vf.to(tdt)
        ksc = vsc = None
        K64, V64 = kst.double(), vst.double()
    del kf, vf
    done = torch.zeros(B, dtype=torch.int32, device="cuda")
    if W > 2:
        done[kv_div:2 * kv_div] = 1          # window 1 has ended (all its beams)
    out = torch.full((B, dm), 7.0, device="cuda", dtype=tdt)
    torch.cuda.synchronize()
    _lib.check(toy.lib.wk_test_cross_attention_splitk(toy.handle, p(part), splits, Bp, p(bq), p(kst), p(vst), p(ksc), p(vsc), p(out), B, H, T,
                                                      wdt, p(done), kv_div))
    torch.cuda.synchronize()
    live = (done == 0).cpu()
    assert torch.all(out[~live.cuda()].float() == 7.0), "a done row was written"
    pv = part[:, :B].double()
    q = (bq.double() + pv.sum(0)).view(B, H, 64)
    qmag = (bq.double().abs() + pv.abs().sum(0)).view(B, H, 64)
    valid = torch.ones(1, 1, T, dtype=torch.bool, device="cuda")
    worst_err, worst_ratio = 0.0, 0.0
    for w0 in range(0, W, 8):                 # 8 windows at a time: the float64 K/V of all 160 rows would take ~5 GB
        w1 = min(W, w0 + 8)
        r0, r1 = w0 * kv_div, w1 * kv_div
        Kx = K64[w0:w1].repeat_interleave(kv_div, dim=0)
        Vx = V64[w0:w1].repeat_interleave(kv_div, dim=0)
        ref = attention_ref(q[r0:r1], Kx, Vx, valid)
        bound = attention_bound(q[r0:r1], qmag[r0:r1], splits + 1, Kx, Vx, valid, ref, dt, hilo=kv_div > 1)
        err = (out[r0:r1].view(r1 - r0, H, 64).double() - ref).abs()
        lv = live[r0:r1]
        if lv.any():
            e, b = err[lv.cuda()], bound[lv.cuda()]
            bad = int((~(e <= b)).sum().item())
            assert bad == 0, f"rows {r0}..{r1}: {bad} elements outside the bound (max err {e.max().item():.3e})"
            worst_err, worst_ratio = max(worst_err, e.max().item()), max(worst_ratio, (e / b).max().item())
    print(f"[cross-attention {dt} d {d} B {B} kv_div {kv_div} fp8 {fp8} splits {splits}] worst error {worst_err:.3e}, "
          f"{worst_ratio:.3f} of its bound")


# ================================================================================== 3. end to end at the benchmarked row counts
@pytest.mark.parametrize("policy", ["bf16", "f16"])
def test_greedy_130_windows_in_one_session(policy):
    """130 windows in one session at large-v3 widths (d 1280, 20 heads, vocabulary 51866; 1 encoder and 2 decoder layers): Bp = 144, so every
    decoder GEMM runs 256-column tiles with 112 zero-filled columns.  Six teacher-forced steps of rows at the edges of the 16-row groups and
    of the 64- and 128-row marks match the same-policy oracle twin (each row alone on the CPU, from that window's own cross K/V), and a
    20-step greedy decode of each of those rows equals its window decoded alone."""
    B = 130
    rows = [0, 15, 16, 63, 64, 127, 128, 129]
    cfg = dict(enc_layers=1, dec_layers=2)
    dims = dataclasses.replace(M.VARIANTS["large-v3"], **cfg)
    w = M.random_weights(dims, seed=41, policy=policy)
    model = wk.Model("large-v3", max_batch=B, dtype=policy, config=cfg)
    model.load_state_dict(w)
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, B)
    pcm = np.stack([mel_ref.synthetic_pcm(2000 + i) for i in range(B)]).astype(np.float32)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    enc_rows = enc_t.numpy()[rows]
    orc = M.WhisperOracle(dims, w, policy)
    dec.bindEncoderOutput(enc_t)
    dec.prepareDecoderInputs()
    worst = np.zeros(len(rows))
    with torch.no_grad():
        cross = orc.cross_kv(torch.from_numpy(enc_rows).transpose(1, 2).contiguous())
        cache = orc.new_cache(len(rows))
        rng = np.random.default_rng(6)
        for pos in range(6):
            toks = rng.integers(0, dims.vocab, size=B)
            lg = dec.predictLogits(toks, [pos] * B)
            ref = orc.decode_step(torch.from_numpy(toks[rows]), pos, cache, cross).numpy()
            for i, r in enumerate(rows):
                worst[i] = max(worst[i], rel_err(lg[r], ref[i]))
    print(f"[130 windows/{policy}] 6 teacher-forced steps, logits rel err vs the same-policy oracle per row {dict(zip(rows, np.round(worst, 6)))} "
          f"(tolerance {TOL_TWIN[policy]:.0e})")
    assert (worst <= TOL_TWIN[policy]).all(), worst
    # a different forced text token per window (prefixTokens), so that rows decode differently and a mix-up of rows cannot go unnoticed
    st = wk.SpecialTokens(**LV3)
    kw = dict(firstTokenLogProbThreshold=None, sampleLength=20, temperatureFallbackCount=0)
    opts = [wk.DecodingOptions(prefixTokens=[1000 + 211 * i], **kw) for i in range(B)]
    prompts = [dec.prefillDecoderInputs(o, st) for o in opts]
    res = dec.decodeText(enc_t, prompts, opts, st)
    assert all(r.steps == 20 or r.tokens[-1] == st.endToken for r in res)
    continuations = {tuple(r.tokens[len(prompts[i]):]) for i, r in enumerate(res)}
    print(f"[130 windows/{policy}] distinct continuations after the prompts among the 130 windows: {len(continuations)}")
    assert len(continuations) > 1
    one = wk.TextDecoder(model, 1)
    for r in rows:
        r1 = one.decodeText(enc.encodeFeatures(fe.logMelSpectrogram(pcm[r:r + 1])), prompts[r], opts[r], st)[0]
        assert r1.tokens == res[r].tokens, (r, r1.tokens, res[r].tokens)
        np.testing.assert_allclose(r1.tokenLogProbs, res[r].tokenLogProbs, atol=1e-5)
    one.close()
    dec.close()
    model.close()


def test_beam5_32_windows_160_rows():
    """32 windows x 5 beams = 160 decode rows in one session (Bp = 160: 256-column tiles, the beam cross-attention kernel with 5 rows per
    K/V block, cache ancestry across 160 rows), at toy128 width.  Every window's result equals the window decoded alone, and the first and
    last windows match oracle.beam_ref.decode_text_beam driven by the GPU's own logits (f16 policy: log-probs to 5e-4, see test_gpu_beam)."""
    beam, n_win = 5, 32
    st_o = D.SpecialTokens.toy(2048)
    st = wk.SpecialTokens.from_any(st_o)
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="toy128", maxBatch=beam * n_win, seed=19, specialTokens=st, dtype="f16"))
    pcm = np.stack([mel_ref.synthetic_pcm(3000 + i) for i in range(n_win)])
    kw = dict(firstTokenLogProbThreshold=None, sampleLength=22, temperatureFallbackCount=0, logProbThreshold=None,
              compressionRatioThreshold=None)
    # a different forced text token per window (prefixTokens), so that windows decode differently
    prefix = [[10 + 31 * b] for b in range(n_win)]
    o_gpu = [wk.DecodingOptions(beamSize=beam, prefixTokens=prefix[b], **kw) for b in range(n_win)]
    res = kit.transcribe(pcm, o_gpu)
    assert len(res) == n_win
    for b in range(n_win):
        alone = kit.transcribe(pcm[b], o_gpu[b])[0]
        assert alone.tokens == res[b].tokens, (b, alone.tokens, res[b].tokens)
    for b in (0, n_win - 1):
        prompt = kit.textDecoder.prefillDecoderInputs(o_gpu[b], st)
        assert prompt == D.prefill_prompt(D.DecodingOptions(prefixTokens=prefix[b], **kw), st_o, True)
        predict, dec = _predictor(kit.model, pcm[b], beam)
        ref = BR.decode_text_beam(predict, prompt, D.DecodingOptions(prefixTokens=prefix[b], **kw), st_o, True, beam, 1.0)
        dec.close()
        assert res[b].tokens == ref.tokens, (b, res[b].tokens, ref.tokens)
        np.testing.assert_allclose(res[b].tokenLogProbs, ref.tokenLogProbs, atol=5e-4)
        assert abs(res[b].avgLogProb - ref.avgLogProb) < 5e-4 and res[b].steps == ref.steps
    distinct = len({tuple(r.tokens) for r in res})
    print(f"[beam 5 x 32 windows] distinct token sequences: {distinct} of {n_win}")
    assert distinct > 1
