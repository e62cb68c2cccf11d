"""The MX fp8 forward path (``Solver.use_fp8_mlp``) against an exact oracle: quantiser, GEMM and MLP layer.

* **Encoder.**  ``scale_exp_oracle`` / ``e4m3_oracle`` are written here from the definitions, in integer
  arithmetic: the scale exponent is the smallest e with amax * 2^-e <= 448, clamped to [-127, 127]; an element
  is x * 2^-e rounded to nearest even on the e4m3 grid (3 fraction bits, subnormals 2^-9 apart), saturated at
  448.  A CPU test holds the oracle against torch's float8 cast and against the product's host mirrors.
* **Quantiser kernels.**  ``mx_quantize`` and the serving ``quantize_rows`` are bit-exact to the oracle, at
  block magnitudes over the whole fp32 exponent range, including blocks whose amax lies below 448 * 2^-126 and
  fp32-subnormal elements.
* **GEMM.**  Every operand is an e4m3 value times a power of two, so fp64 of the dequantised operands is exact.
  With one nonzero product per output the kernel's result is exact too, and every scale byte read from the wrong
  row, column, slice or k-block is a bit mismatch.  General data is held to
  ``r |ref| + alpha (C_MMA + (slices + 2) 2^-24) sum|a_q b_q| + 2^-24 |bias|``: r the output rounding,
  C_MMA the error of one m64n128k32 e4m3 wgmma over its 32 products relative to their magnitude sum
  (measured below), and one fp32 rounding per slice promotion, alpha and bias.
* **Layer.**  ``MLPLayer`` with ``use_fp8_mlp`` at the bench's MLPs: each fp8 GEMM against fp64 of the
  oracle-quantised bf16 input and weights, the bf16 layers against the bf16 GEMM bound, and the backward (bf16,
  straight-through: unquantised weights) against fp64 on the forward's own activations.
"""
import functools
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_dense_path_fp64_gpu as DP  # noqa: E402
from hugectr_b200.ops import gemm as G  # noqa: E402
from hugectr_b200.ops import mxfp8 as MX  # noqa: E402

f64, i64 = torch.float64, torch.int64
U = 2.0 ** -24
F32_R = 2.0 ** -23
FP32_MIN_NORMAL = 2.0 ** -126
E4M3_MAX_CODE = 0x7E          # 448
gpu = pytest.mark.gpu
DEV = "cuda"

# Error of one m64n128k32 e4m3 wgmma (fp32 output) against the exact sum of its 32 products, relative to the sum
# of their magnitudes: the largest value test_c_mma_one_slice measured on an H100 80GB HBM3 (700 W) was
# 7.805e-4 = 2^-10.32, over 1M outputs of 32 products with random signs and codes over the whole e4m3 range.  The
# bound takes it with a 2x margin.
C_MMA_MEASURED = 7.805e-4
C_MMA = 2 * C_MMA_MEASURED


# ============================================================================ oracle
def scale_exp_oracle(amax):
    """int64 exponents: the smallest e with amax * 2^-e <= 448, clamped to [-127, 127]; -127 for amax == 0"""
    a = amax.to(f64)
    _, ex = torch.frexp(a)                                   # a = m 2^ex, m in [0.5, 1): the answer is ex-9 or ex-8
    e = ex.to(i64) - 9
    e = e + (a > 448.0 * torch.exp2(e.to(f64))).to(i64)
    ok = (a == 0) | (a <= 448.0 * torch.exp2(e.to(f64))) & (a > 448.0 * torch.exp2((e - 1).to(f64)))
    assert bool(ok.all())
    return torch.where(a > 0, e, torch.full_like(e, -127)).clamp(-127, 127)


def e4m3_oracle(x, e):
    """uint8 e4m3 codes of x * 2^-e (x fp32 / bf16, e int64 broadcastable), rounded to nearest even, saturated"""
    x = x.to(f64)
    mx, E = torch.frexp(x)                                   # x = mx 2^E exactly, |mx| in [0.5, 1)
    M = (mx.abs() * 2.0 ** 24).to(i64)                       # x = +-M 2^(E - 24), M < 2^24 an integer
    E = E.to(i64)
    k = E - 1 - e                                            # |x 2^-e| in [2^k, 2^(k+1))
    qe = torch.clamp(k - 3, min=-9)                          # grid spacing 2^qe: 3 fraction bits, subnormals 2^-9
    s = (qe - (E - 24 - e)).clamp(1, 62)                     # >= 20 always: M 2^(E-24-e) / 2^qe = M >> s
    q0 = M >> s
    rem = M - (q0 << s)
    half = torch.ones_like(s) << (s - 1)
    q = q0 + ((rem > half) | ((rem == half) & (q0 & 1 == 1))).to(i64)
    up = q == 16                                             # rounded up into the next binade
    q = torch.where(up, torch.full_like(q, 8), q)
    qe = qe + up.to(i64)
    code = torch.where((qe == -9) & (q < 8), q, ((qe + 10) << 3) + q - 8)
    code = torch.where(M == 0, torch.zeros_like(code), code).clamp(max=E4M3_MAX_CODE)
    return (code | (torch.signbit(x).to(i64) << 7)).to(torch.uint8)


def mx_oracle(x):
    """x [rows, cols] -> (codes [rows, cols] uint8, scale bytes [rows, cols / 32] uint8)"""
    rows, cols = x.shape
    blk = x.reshape(rows, cols // 32, 32)
    e = scale_exp_oracle(blk.float().abs().amax(-1))
    return e4m3_oracle(blk, e.unsqueeze(-1)).reshape(rows, cols), (e + 127).to(torch.uint8)


def sf_index(rows_pad, cols):
    """flat index into the kernel's scale array of each (row, 32-wide block):
    [r / 128][k / 128][r % 32][(r % 128) / 32][(k % 128) / 32]"""
    r = torch.arange(rows_pad).view(-1, 1)
    k = torch.arange(cols // 32).view(1, -1) * 32
    return ((r // 128) * (cols // 128) + k // 128) * 512 + (r % 32) * 16 + ((r % 128) // 32) * 4 + (k % 128) // 32


def decode(codes):
    return codes.view(torch.float8_e4m3fn).to(f64)


def dequant(codes, sbytes):
    """fp64 values of codes [rows, cols] with scale bytes [rows, cols / 32] (exact)"""
    rows, cols = codes.shape
    sc = torch.exp2(sbytes.to(f64) - 127.0)
    return (decode(codes).view(rows, cols // 32, 32) * sc.unsqueeze(-1)).view(rows, cols)


def kernel_scales(sf, rows, cols):
    """scale bytes [rows, cols / 32] read out of the kernel's block layout by ``sf_index``"""
    return sf.cpu()[sf_index(MX._pad128(rows), cols)][:rows]


# ============================================================================ CPU: the oracle itself
def _finite_codes():
    c = torch.arange(256, dtype=torch.uint8)
    return c[(c & 0x7F) != 0x7F]


def test_oracle_codes_and_midpoints_cpu():
    """every e4m3 code encodes to itself; every midpoint between neighbouring codes rounds to the even code, as
    torch's float8 cast does; values above 448 saturate"""
    codes = _finite_codes()
    v = decode(codes).float()
    assert torch.equal(e4m3_oracle(v, torch.zeros((), dtype=i64)), codes)
    pos = torch.arange(0, E4M3_MAX_CODE + 1, dtype=torch.uint8)
    pv = decode(pos)
    mid = ((pv[:-1] + pv[1:]) / 2).float()                   # exact in fp32
    for sgn in (1.0, -1.0):
        got = e4m3_oracle(sgn * mid, torch.zeros((), dtype=i64))
        assert torch.equal(got, (sgn * mid).to(torch.float8_e4m3fn).view(torch.uint8))
        assert bool(((got & 1) == 0).all())                  # ties to the even code
    for s in (0, 3, -40, 100):                               # the same grid at any scale
        e = torch.full((), s, dtype=i64)
        assert torch.equal(e4m3_oracle((v.to(f64) * 2.0 ** s).float(), e), codes)
    big = torch.tensor([448.0, 449.0, 463.9, 464.0, 480.0, 1e4, 3e38, -1e4])
    assert torch.equal(e4m3_oracle(big, torch.zeros((), dtype=i64)),
                       torch.tensor([0x7E] * 7 + [0xFE], dtype=torch.uint8))


def _all_finite_bf16():
    b = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).float()
    return b[torch.isfinite(b)]


def test_oracle_matches_host_mirrors_on_every_bf16_cpu():
    """every finite bf16 value, in 32-wide blocks of several amax: the oracle against mx_quantize_reference (q and
    the scale bytes in their block layout) and against the serving rule fp8_rows_quantize"""
    from hugectr_b200.embedding import ops as E
    vals = _all_finite_bf16()
    n = vals.numel() // 128 * 128
    g = torch.Generator().manual_seed(0)
    layouts = [vals[:n], vals[torch.randperm(vals.numel(), generator=g)[:n]]]
    for k in (-133, -126, -100, 0, 1, 60):                   # a block amax of exactly 448 * 2^k beside every value
        x = vals[torch.randperm(vals.numel(), generator=g)[:n]].clone().view(-1, 32)
        x = x * (x.abs() <= 448.0 * 2.0 ** k)
        x[:, 0] = 448.0 * 2.0 ** k
        layouts.append(x.reshape(-1))
    for x in layouts:
        x = x.view(-1, 128)
        q, s = mx_oracle(x)
        qr, sfr = MX.mx_quantize_reference(x)
        assert torch.equal(qr[:x.shape[0]], q)
        assert torch.equal(sfr[sf_index(x.shape[0], 128)], s)
        qs, es = E.fp8_rows_quantize(x.view(-1, 32))
        assert torch.equal(qs.view(torch.uint8), q.view(-1, 32))
        assert torch.equal(es, s.view(-1))


def test_scale_exponent_every_fp32_significand_cpu():
    """the host scale rule (integer form) against the definition on every fp32 significand, at exponents across
    the range, and on fp32 subnormals"""
    m = torch.arange(1 << 23, dtype=torch.int32)
    for biased in (1, 2, 7, 8, 9, 100, 127, 135, 136, 254):
        a = (m | (biased << 23)).view(torch.float32)
        assert torch.equal(MX.e4m3_scale_exponent(a).to(i64), scale_exp_oracle(a))
    a = m[::97].view(torch.float32)                          # subnormals and zero
    assert torch.equal(MX.e4m3_scale_exponent(a).to(i64), scale_exp_oracle(a))


# ============================================================================ GEMM guards (predicate only)
def test_gemm_mxfp8_eligible_cpu():
    M, N, K = 200, 64, 256
    aq, sfa = MX.mx_buffers(M, K, "cpu")
    bq, sfb = MX.mx_buffers(N, K, "cpu")
    out = torch.empty(M, N, dtype=torch.bfloat16)
    bias = torch.zeros(N)
    ok = MX.gemm_mxfp8_eligible
    assert ok(aq, sfa, bq, sfb, M, N, K, out, bias, G.EPI_RELU)
    assert ok(aq, sfa, bq, sfb, M, N, K, torch.empty(M, N), bias, G.EPI_OUT_F32 | G.EPI_SIGMOID)
    for f in (G.EPI_MASK, G.EPI_CROSS, G.EPI_ADD, G.EPI_ATOMIC):
        assert not ok(aq, sfa, bq, sfb, M, N, K, out, bias, f)
    assert not ok(aq, sfa, bq, sfb, M, N, K, torch.empty(M, N), bias, 0)           # fp32 out without OUT_F32
    assert not ok(aq, sfa, bq, sfb, M, N, 200, out, bias, 0)                      # K % 128
    wide = torch.empty(M, N + 1, dtype=torch.bfloat16)
    assert not ok(aq, sfa, bq, sfb, M, N, K, wide[:, :N], bias, 0)                # 2-byte row pitch misaligned
    assert not ok(aq, sfa, bq, sfb, M, N, K, wide.view(-1)[1:1 + M * N].view(M, N), bias, 0)   # base misaligned
    assert not ok(aq, sfa, bq, sfb, M, N, K, out, torch.zeros(N + 1)[1:], 0)     # bias base misaligned
    assert not ok(aq, sfa, bq, sfb, M, N, K, out, torch.zeros(N - 1), 0)         # bias too short
    assert not ok(aq[:-1], sfa, bq, sfb, M, N, K, out, bias, 0)                  # fewer rows than the tensor map
    assert not ok(aq, sfa, bq[:-1], sfb, M, N, K, out, bias, 0)
    assert not ok(aq, sfa[:-16], bq, sfb, M, N, K, out, bias, 0)                 # fewer scale bytes than copied
    assert not ok(aq, sfa, bq, sfb[:-16], M, N, K, out, bias, 0)
    shifted = lambda t: torch.zeros(t.numel() + 16, dtype=torch.uint8)[1:1 + t.numel()]  # noqa: E731
    assert not ok(aq, shifted(sfa), bq, sfb, M, N, K, out, bias, 0)              # bases not 16-byte aligned
    assert not ok(aq, sfa, shifted(bq).view(bq.shape), sfb, M, N, K, out, bias, 0)
    assert ok(aq, sfa, bq, sfb, M, 16, K, out[:, :16], None, 0)                   # N < 32: scalar epilogue


# ============================================================================ quantiser kernels (bit-exact)
@functools.lru_cache(maxsize=16)       # every (rows, cols) of the quantiser test, reused by its 4 variants
def mx_input(rows, cols, seed):
    """fp32 [rows, cols]: 32-wide blocks with magnitudes log-uniform over the whole fp32 range, and the rule's
    edge blocks in turn"""
    g = torch.Generator().manual_seed(seed)
    nb = rows * cols // 32
    x = torch.randn(nb, 32, generator=g) * torch.exp2(torch.rand(nb, 1, generator=g) * 270 - 150)
    kk = torch.randint(-120, 120, (nb,), generator=g).to(f64)
    top = 448.0 * torch.exp2(kk)
    lanes = torch.randint(0, 32, (nb,), generator=g)
    frac = torch.rand(nb, 32, generator=g).to(f64)
    for b in range(nb):
        t, k, a = b % 16, int(kk[b]), float(top[b])
        row = None
        if t == 0:                                          # amax exactly 448 * 2^k, then its fp32 neighbours
            row = frac[b] * a
        elif t in (1, 2):
            a = torch.nextafter(torch.tensor(a, dtype=torch.float32),
                                torch.tensor(math.inf if t == 1 else 0.0)).item()
            row = frac[b] * a
        elif t == 3:                                        # all zero
            row = torch.zeros(32, dtype=f64)
        elif t == 4:                                        # one nonzero element
            row = torch.zeros(32, dtype=f64)
            a = -a if b % 3 == 0 else a
        elif t == 5:                                        # negative
            row = -frac[b] * a
            a = -a
        elif t == 6:                                        # scaled results that are e4m3 subnormals, and ties
            j = torch.randint(0, 16, (32,), generator=g).to(f64)
            row = j * 2.0 ** -10 * 2.0 ** k
        elif t == 7:                                        # exact ties on the normal grid
            m = torch.randint(0, 8, (32,), generator=g).to(f64)
            p = torch.randint(-6, 8, (32,), generator=g).to(f64)
            row = (8 + m + 0.5) / 8 * torch.exp2(p) * 2.0 ** k
        elif t == 8:                                        # amax in [2^-126, 448 * 2^-126): flush band
            a = 2.0 ** -126 * (1 + 447 * float(frac[b, 0]))
            row = frac[b] * a
        elif t == 9:                                        # fp32-subnormal elements under a flush-band amax
            a = 2.0 ** -119
            row = torch.exp2(-149 + frac[b] * 22)
        elif t == 10:                                       # all elements fp32-subnormal
            row = torch.exp2(-149 + frac[b] * 22) * torch.sign(torch.randn(32, generator=g))
            a = None
        if row is not None:
            x[b] = row.float()
            if a is not None:
                x[b, lanes[b]] = a
    return x.view(rows, cols)


def _stored(x, dtype, transposed, pad=24):
    """x [rows, cols] on the device in ``dtype``, row-major or transposed ([cols, rows]), pitch > width"""
    src = x.t() if transposed else x
    base = torch.zeros(src.shape[0], src.shape[1] + pad, dtype=dtype, device=DEV)
    base[:, :src.shape[1]] = src.to(dtype).to(DEV)
    return base[:, :src.shape[1]]


@gpu
@pytest.mark.parametrize("cols", [128, 384, 3456])
@pytest.mark.parametrize("rows", [1, 127, 128, 129, 300])
@pytest.mark.parametrize("transposed", [False, True], ids=["rowmajor", "transposed"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_mx_quantize_kernel_bit_exact(dtype, transposed, rows, cols):
    x = mx_input(rows, cols, rows * 7 + cols)
    xs = _stored(x, dtype, transposed)
    q, sf = MX.mx_buffers(rows, cols, DEV)
    q.fill_(0xAB)
    sf.fill_(0xAB)
    MX.mx_quantize(xs, q, sf, transposed=transposed)
    want_q, want_s = mx_oracle(x.to(dtype).float())
    q = q.cpu()
    rp = MX._pad128(rows)
    bad = (q[:rows] != want_q).nonzero()
    assert bad.numel() == 0, (f"{bad.shape[0]} codes differ, first at {tuple(bad[0].tolist())}: got "
                              f"{int(q[tuple(bad[0])])} want {int(want_q[tuple(bad[0])])} x={x[tuple(bad[0])]!r}")
    assert torch.equal(kernel_scales(sf, rows, cols), want_s)
    assert bool((q[rows:] == 0).all())                                   # padding rows: zero, scale 2^-127
    assert bool((sf.cpu()[sf_index(rp, cols)][rows:] == 0).all())


@gpu
@pytest.mark.parametrize("pitch", [7, 64])
def test_serving_quantize_rows_tiny_amax(pitch):
    """hctr_emb_quantize_rows on rows whose amax lies below 448 * 2^-126 or whose elements are fp32 subnormals"""
    from hugectr_b200.embedding import ops as E
    g = torch.Generator().manual_seed(pitch)
    amax = torch.tensor([2.0 ** -126, 2.0 ** -120, 447.0 * 2.0 ** -126, 2.0 ** -127, 2.0 ** -140, 448 * 2.0 ** -126,
                         1.0])
    x = (torch.rand(len(amax), pitch, generator=g) * 2 - 1) * amax.unsqueeze(1)
    x[:, 0] = amax
    x[3:5] = torch.exp2(-149 + torch.rand(2, pitch, generator=g) * 22)   # fp32-subnormal rows
    x[1, 1:] = torch.exp2(-149 + torch.rand(pitch - 1, generator=g) * 22)
    n = x.shape[0]
    table = torch.full((n * pitch,), 0x55, dtype=torch.uint8, device=DEV).view(torch.float8_e4m3fn)
    exps = torch.zeros(n, dtype=torch.uint8, device=DEV)
    bad = torch.zeros(1, dtype=torch.int32, device=DEV)
    E.quantize_rows(x, torch.arange(n), table, exps, bad)
    e = scale_exp_oracle(x.abs().amax(1))
    assert int(bad.item()) == 0
    assert torch.equal(exps.cpu(), (e + 127).to(torch.uint8))
    assert torch.equal(table.view(torch.uint8).view(n, pitch).cpu(), e4m3_oracle(x, e.unsqueeze(1)))


# ============================================================================ GEMM
ONE = 0x38                    # e4m3 code of 1.0


def _nonzero_codes(shape, g):
    """random finite nonzero e4m3 codes of both signs"""
    c = torch.randint(1, 0x7F, shape, generator=g).to(torch.uint8)
    return c | (torch.randint(0, 2, shape, generator=g).to(torch.uint8) << 7)


def _pack(codes, sbytes):
    """(q [rows_pad, K] on the device, sf in the block layout) of codes [rows, K] and scale bytes [rows, K / 32];
    padding rows hold codes (the kernel must not store their outputs) and scale byte 127"""
    rows, K = codes.shape
    rp = MX._pad128(rows)
    q = torch.full((rp, K), ONE, dtype=torch.uint8)
    q[:rows] = codes
    s = torch.full((rp, K // 32), 127, dtype=torch.uint8)
    s[:rows] = sbytes
    sf = torch.zeros(rp // 128 * (K // 128) * 512, dtype=torch.uint8)
    sf[sf_index(rp, K)] = s
    return q.to(DEV), sf.to(DEV)


def _out_buf(M, N, dtype):
    """out [M, N] view of a NaN-filled [M + 4, ldo] buffer, ldo > N with 16-byte rows (rows M.. and columns N..
    must stay NaN)"""
    base = torch.full((M + 4, (N + 8) // 8 * 8 + 8), float("nan"), dtype=dtype, device=DEV)
    return base, base[:M, :N]


def _assert_untouched(base, M, N):
    assert bool(torch.isnan(base[M:]).all()) and bool(torch.isnan(base[:, N:]).all()), "stored out of bounds"


def _single_product_operands(M, N, K, g):
    """A [M, K], B [N, K] codes with exactly one k where both are nonzero for every (m, n): row m of A covers
    grid row m % 8 of an 8 x 8 grid of k positions, row n of B grid column n % 8.  The 64 positions fill the
    4 slices of the first and the last k-blocks and slices in between.  Scale bytes differ per row and slice."""
    slices = K // 32
    order = [0, 1, 2, 3, slices - 4, slices - 3, slices - 2, slices - 1] + list(range(4, slices - 4))
    order = list(dict.fromkeys(s for s in order if 0 <= s < slices))
    kpos = torch.empty(8, 8, dtype=i64)
    for idx in range(64):
        kpos[idx // 8, idx % 8] = order[idx % len(order)] * 32 + (idx // len(order)) * 5 % 32
    assert kpos.unique().numel() == 64
    a = torch.zeros(M, K, dtype=torch.uint8)
    b = torch.zeros(N, K, dtype=torch.uint8)
    rm, rn = torch.arange(M) % 8, torch.arange(N) % 8
    for m in range(M):
        a[m, kpos[rm[m]]] = _nonzero_codes((8,), g)
    for n in range(N):
        b[n, kpos[:, rn[n]]] = _nonzero_codes((8,), g)
    s = torch.arange(slices).view(1, -1)
    sa = (127 + (torch.arange(M).view(-1, 1) * 5 + s * 3) % 17 - 8).to(torch.uint8)
    sb = (127 + (torch.arange(N).view(-1, 1) * 3 + s * 7) % 19 - 9).to(torch.uint8)
    return a, sa, b, sb


@gpu
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("M,N,K", [(300, 200, 256), (129, 131, 3456), (64, 1, 128), (1, 257, 640)])
def test_gemm_mxfp8_slice_indexing_bit_exact(M, N, K, out_dtype):
    """one nonzero product per output: out = a b 2^(ea + eb - 254) exactly (8 significant bits fit bf16)"""
    g = torch.Generator().manual_seed(M + N + K)
    a, sa, b, sb = _single_product_operands(M, N, K, g)
    aq, sfa = _pack(a, sa)
    bq, sfb = _pack(b, sb)
    base, out = _out_buf(M, N, out_dtype)
    flags = G.EPI_OUT_F32 if out_dtype == torch.float32 else 0
    MX.gemm_mxfp8(aq, sfa, bq, sfb, M, N, K, out=out, flags=flags)
    ref = dequant(a, sa) @ dequant(b, sb).t()
    torch.cuda.synchronize()
    _assert_untouched(base, M, N)
    got = out.cpu().to(f64)
    bad = (got != ref).nonzero()
    assert bad.numel() == 0, (f"{bad.shape[0]} outputs differ, first {tuple(bad[0].tolist())}: got "
                              f"{got[tuple(bad[0])].item()!r} want {ref[tuple(bad[0])].item()!r}")


@gpu
@pytest.mark.parametrize("lo", [False, True], ids=["upper_end", "lower_end"])
def test_gemm_mxfp8_scale_range(lo):
    """one product 1 * 1 (or 448 * 448) per output at scale bytes ea (row), eb (column), the same for every slice:
    exact while c = ea + eb - 254 is in [-126, 127] and neither byte is 0; a zero byte or c < -126 drops the slice
    even where the result would be a normal number; for c > 127 the scale product is +inf, and the slices without a
    product add 0 * inf = NaN (gemm_mxfp8.cu's header)"""
    M = N = 128
    K = 128
    big = lo                                                 # 448 * 448 ~ 2^17.6: 2^c times it is normal to c = -143
    code = 0x7E if big else ONE
    a = torch.zeros(M, K, dtype=torch.uint8)
    b = torch.zeros(N, K, dtype=torch.uint8)
    a[:, 37] = code
    b[:, 37] = code
    r = torch.arange(128)
    ea = (64 + r) if lo else (128 + r)                       # lower end: c in [-190, 64]; upper: [2, 256]
    eb = r if lo else (128 + r)
    sa = ea.to(torch.uint8).view(-1, 1).expand(M, K // 32).contiguous()
    sb = eb.to(torch.uint8).view(-1, 1).expand(N, K // 32).contiguous()
    aq, sfa = _pack(a, sa)
    bq, sfb = _pack(b, sb)
    out = MX.gemm_mxfp8(aq, sfa, bq, sfb, M, N, K, flags=G.EPI_OUT_F32).cpu().to(f64)
    c = (ea.view(-1, 1) + eb.view(1, -1) - 254).to(f64)
    part = 448.0 * 448.0 if big else 1.0
    exact = part * torch.exp2(c)
    inside = (c >= -126) & (c <= 127) & (ea.view(-1, 1) > 0) & (eb.view(1, -1) > 0)
    assert torch.equal(out[inside], exact[inside])
    assert bool(torch.isnan(out[c > 127]).all())
    assert bool((out[~inside & (c <= 127)] == 0).all())
    if lo:                                                   # dropped although the exact result is normal fp32
        assert bool(((~inside) & (exact >= FP32_MIN_NORMAL) & (out == 0)).any())


def _block_scaled(rows, K, g, row_pat, slice_pat):
    """fp32 [rows, K]: randn with a power-of-two magnitude per (row, 32-wide slice), so that the scale bytes
    differ between neighbouring rows, columns and slices; some blocks negative-heavy, a few all zero"""
    s = torch.arange(K // 32).view(1, -1)
    ex = ((torch.arange(rows).view(-1, 1) * row_pat + s * slice_pat) % 13 - 6).float()
    x = torch.randn(rows, K // 32, 32, generator=g) * torch.exp2(ex).unsqueeze(-1)
    x[(torch.arange(rows) % 11 == 3), 1 % (K // 32)] = 0.0
    return x.view(rows, K)


def out_r(dtype):
    return DP.BF16_R if dtype == torch.bfloat16 else U


def acc_bound(mag, slices, alpha=1.0, bias=None):
    """error of the fp32 value the epilogue activates and stores: C_MMA per slice product sum, one rounding per
    slice promotion, alpha and bias"""
    tol = alpha * (C_MMA + (slices + 2) * U) * mag
    if bias is not None:
        tol = tol + U * bias.to(f64).abs().view(1, -1)
    return tol


EPILOGUES = {
    "none": dict(flags=0, bias=False, alpha=1.0, f32=False),
    "bias": dict(flags=0, bias=True, alpha=1.0, f32=False),
    "relu": dict(flags=G.EPI_RELU, bias=True, alpha=1.0, f32=False),
    "sigmoid": dict(flags=G.EPI_SIGMOID, bias=True, alpha=1.0, f32=False),
    "f32_alpha": dict(flags=G.EPI_OUT_F32, bias=True, alpha=0.375, f32=True),
}
SHAPES = [(1, 100, 256), (64, 1, 128), (127, 31, 640), (129, 200, 3456), (1000, 128, 256), (6912, 1024, 3456),
          (129, 1024, 128)]


@gpu
@pytest.mark.parametrize("epi", list(EPILOGUES))
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_mxfp8_general(M, N, K, epi):
    c = EPILOGUES[epi]
    out_dtype = torch.float32 if c["f32"] else torch.bfloat16
    g = torch.Generator().manual_seed(M * 3 + N * 5 + K)
    a = _block_scaled(M, K, g, 5, 3)
    b = _block_scaled(N, K, g, 3, 7) * 0.05
    bias = (torch.randn(N, generator=g) * 0.5).to(DEV) if c["bias"] else None
    aq, sfa = MX.mx_quantize(a.to(DEV))
    bq, sfb = MX.mx_quantize(b.to(DEV))
    base, out = _out_buf(M, N, out_dtype)
    MX.gemm_mxfp8(aq, sfa, bq, sfb, M, N, K, out=out, bias=bias, flags=c["flags"], alpha=c["alpha"])
    A = dequant(aq.cpu()[:M], kernel_scales(sfa, M, K)).to(DEV)
    B = dequant(bq.cpu()[:N], kernel_scales(sfb, N, K)).to(DEV)
    ref = c["alpha"] * (A @ B.t())
    mag = A.abs() @ B.abs().t()
    if bias is not None:
        ref = ref + bias.to(f64).view(1, -1)
    tol = acc_bound(mag, K // 32, c["alpha"], bias)
    if c["flags"] & G.EPI_RELU:
        ref = torch.relu(ref)
    if c["flags"] & G.EPI_SIGMOID:
        # sigmoid is 1/4-Lipschitz; 1 / (1 + __expf(-v)): __expf's documented error of 2 + floor(1.173 |v|) ulp is
        # relative to its value and perturbs the sigmoid by at most that relative amount; the fast division and
        # the addition add 2.5 ulp
        v = ref
        ref = torch.sigmoid(v)
        tol = tol / 4 + (5 + torch.floor(1.173 * v.abs())) * F32_R * ref + FP32_MIN_NORMAL
    r = out_r(out_dtype)
    tol = r * ref.abs() + (1 + r) * tol
    torch.cuda.synchronize()
    _assert_untouched(base, M, N)
    DP.assert_bound(out, ref, tol, f"gemm_mxfp8 {epi}")


@gpu
def test_c_mma_one_slice():
    """one full 32-wide slice per output (all other slices zero, every scale 2^0): the measured error of one
    e4m3 wgmma against the exact sum of its 32 products, relative to their magnitude sum, stays within C_MMA"""
    M, N, K = 1024, 1024, 256
    g = torch.Generator().manual_seed(9)
    a = torch.zeros(M, K, dtype=torch.uint8)
    b = torch.zeros(N, K, dtype=torch.uint8)
    a[:, 160:192] = _nonzero_codes((M, 32), g)
    b[:, 160:192] = _nonzero_codes((N, 32), g)
    ones_a = torch.full((M, K // 32), 127, dtype=torch.uint8)
    ones_b = torch.full((N, K // 32), 127, dtype=torch.uint8)
    aq, sfa = _pack(a, ones_a)
    bq, sfb = _pack(b, ones_b)
    out = MX.gemm_mxfp8(aq, sfa, bq, sfb, M, N, K, flags=G.EPI_OUT_F32).to(f64)
    A, B = decode(a).to(DEV), decode(b).to(DEV)
    ref, mag = A @ B.t(), A.abs() @ B.abs().t()
    ratio = ((out - ref).abs() / mag).max().item()
    print(f"c_mma measured: {ratio:.3e} = 2^{math.log2(ratio) if ratio > 0 else float('-inf'):.2f}")
    assert ratio <= C_MMA, ratio


# ============================================================================ layer
def _build_fp8_mlp(batch, k, in_dtype, kw):
    from hugectr_b200.enums import Layer_t
    from hugectr_b200.layers import LAYER_REGISTRY, BuildCtx, ParamArena, TensorBag
    from hugectr_b200.solver import CreateSolver, DenseLayer
    dev = torch.device(DEV)
    arena = ParamArena()
    ctx = BuildCtx(arena, dev, torch.bfloat16, batch, True, CreateSolver(use_mixed_precision=True, use_fp8_mlp=True), True)
    x = TensorBag("in0", (batch, k), in_dtype)
    x.data = torch.zeros((batch, k), dtype=in_dtype, device=dev)
    x.grad = torch.zeros((batch, k), dtype=in_dtype, device=dev)
    layer = LAYER_REGISTRY[Layer_t.MLP](DenseLayer(Layer_t.MLP, ["in0"], ["out"], **kw), [x], ctx)
    arena.finalize(dev, True)
    layer.allocate()
    arena.init_params(3)
    g = torch.Generator().manual_seed(5)
    for p in layer.params:
        if p.w.dim() == 2 and p.w.shape[0] == 1:
            p.w.copy_(torch.rand(p.w.shape, generator=g).mul_(0.2).sub_(0.1).to(DEV))
    arena.sync_shadow()
    return layer, x, arena


def _check_fp8_fprop(layer, fp8_layers):
    h = layer._x_in
    for i in range(len(layer.dims_out)):
        bias = None if layer.B[i] is None else layer.B[i].w.reshape(-1)
        W = layer.W[i].w16[:h.shape[1]]
        if i in fp8_layers:
            qa, sa = mx_oracle(h)
            qb, sb = mx_oracle(W.t())
            A, B = dequant(qa, sa), dequant(qb, sb)
            ref, mag = A @ B.t(), A.abs() @ B.abs().t()
            if bias is not None:
                ref = ref + bias.to(f64)
            if layer.relu[i]:
                ref = torch.relu(ref)
            tol = DP.BF16_R * ref.abs() + (1 + DP.BF16_R) * acc_bound(mag, h.shape[1] // 32, 1.0, bias)
            DP.assert_bound(layer.acts[i], ref, tol, f"fp8 acts[{i}]")
        else:
            if layer.dims_out[i] == 1:
                ref, mag = DP.gemm_oracle(h[:, :layer.W[i].shape[0]], layer.W[i].w.reshape(-1, 1), bias=bias)
            else:
                ref, mag = DP.gemm_oracle(h, W, bias=bias)
            if layer.relu[i]:
                ref = torch.relu(ref)
            DP.assert_sum(layer.acts[i], ref, mag, h.shape[1], DP.BF16_R, f"bf16 acts[{i}]")
        h = layer.acts[i]


MLP_CASES = {   # fp8: the layers whose K is a multiple of 128 and whose N is not 1
    "bottom": dict(k=13, in_dtype=torch.float32, in_scale=2.0, fp8={1, 2},
                   kw=dict(num_outputs=[512, 256, 128], act_type="relu")),
    "top": dict(k=3456, in_dtype=torch.bfloat16, in_scale=1.0, fp8={0, 1, 2, 3},
                kw=dict(num_outputs=[1024, 1024, 512, 256, 1], activations=["relu"] * 4 + ["none"])),
}


@gpu
@pytest.mark.parametrize("batch", [6912, 1000])
@pytest.mark.parametrize("which", list(MLP_CASES))
def test_mlp_layer_fp8(which, batch):
    c = MLP_CASES[which]
    kw = dict(c["kw"])
    if "act_type" in kw:
        kw["act_type"] = DP._acts([kw["act_type"]])[0]
    else:
        kw["activations"] = DP._acts(kw["activations"])
    layer, x, arena = _build_fp8_mlp(batch, c["k"], c["in_dtype"], kw)
    for seed in (100, 200):                  # the second pass reuses the layer's fp8 buffers
        DP._feed(layer, x, arena, seed, c["in_scale"])
        layer.fprop(True)
        layer.bprop()
        torch.cuda.synchronize()
        assert set(layer._fp8_bufs) == c["fp8"]
        _check_fp8_fprop(layer, c["fp8"])
        DP.check_mlp_bprop(layer, x)
