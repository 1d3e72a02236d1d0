"""An integer-exact statement of the FP8 export's arithmetic (DESIGN §5.19), and the CPU tests that make it trustworthy.

The contract, for a block of a 2-D F32 / F16 / BF16 weight and its elements x:
  a = the integer max of the bits of |x| widened to F32 (any NaN wins), then max(a, fl32(1e-4)) unless a is a NaN;
  s = RN(a * RN(1 / 448));  m = RN(RN(1 / a) * 448), from a and never from s;
  q = E4M3(RN(x * m)): the exact product rounded to nearest even F32 (subnormals kept), then that F32 value rounded to
      nearest even E4M3 (subnormals down to 2^-9, the sign kept on zeros), saturating: every |y| >= 448 and +-inf give
      0x7E / 0xFE; a NaN product gives 0x7F (the GPU's NaN is positive, so negative NaNs and inf * 0 give 0x7F too).

``reference_block_scales``, ``reference_multiplier`` and ``reference_quant`` use int64 tensor arithmetic only -- no
float type is formed -- so they are independent of the ``FMUL``, ``MUFU.RCP`` and ``cvt`` instructions the kernels and
torch issue, and they run unchanged on CPU and CUDA tensors (tests/test_fp8_quant_paths_gpu.py runs them on the
device).  Products of two F32 significands have 48 bits, so the rounding here takes significands below 2^61, where
the helpers of tests/test_fp8_reference_cpu.py stop at 2^32.

They are checked against torch's CPU model of the export (tests/test_device_file_fp8_cpu.py) for every F16 and BF16
pattern times every structured a, and for the structured and random F32 sets; against a plain ``fractions.Fraction``
rounding on sampled pairs of every class, the saturating region included (c10's conversion gives NaN there); and
against hand-written values.  The coverage test shows that the sets hold pairs of every class, and that four wrong
forms of the arithmetic each give other bits on them."""
import random
from fractions import Fraction

import numpy as np
import torch

from tests.test_cast_reference_cpu import NAN, reference_cast
from tests.test_fp8_reference_cpu import _decode, _fraction_round, _fraction_value

F32, F16, BF16, E4M3 = torch.float32, torch.float16, torch.bfloat16, torch.float8_e4m3fn
F32_FMT, E4M3_WIDE = (8, 23, 127), (5, 3, 7)  # E4M3 rounded with one more exponent bit, then saturated at 0x7E
FLOOR = 0x38D1B717  # fl32(1e-4)
F32_NAN = 0x7FFFFFFF  # the NaN of FMUL and of cvt.f32.f16 on the H100 (NAN_POLICY of the other device tests)
FLT_MAX, F32_INF = 0x7F7FFFFF, 0x7F800000
E4M3_MAX, E4M3_NAN = 0x7E, 0x7F


def _log2(m):
    """floor(log2(m)) for 1 <= m < 2^63 (0 for m = 0)."""
    p = torch.zeros_like(m)
    for k in (32, 16, 8, 4, 2, 1):
        p = torch.where((m >> (p + k)) != 0, p + k, p)
    return p


def _split(m, e, fmt):
    """Rounding m * 2^e (0 < m < 2^61) to a format (ne, nm, bias): (q, kept, rem, half, dn) as in
    tests/test_fp8_reference_cpu.py, for wider significands: 62 dropped bits leave the tie bit above any m < 2^61."""
    _, nm, bias = fmt
    q = torch.clamp(_log2(m) + e, min=1 - bias) - nm
    r = q - e
    dn = torch.clamp(r, 0, 62)
    kept = (m << torch.clamp(-r, min=0)) >> dn
    rem = m & ((torch.ones_like(m) << dn) - 1)
    half = torch.where(dn > 0, torch.ones_like(m) << torch.clamp(dn - 1, min=0), torch.zeros_like(m))
    return q, kept, rem, half, dn


def _round(sign, m, e, fmt):
    """The bits nearest to (-1)^sign * m * 2^e (0 <= m < 2^61) in format fmt, ties to even, subnormals kept, overflow
    to the all-ones exponent with a zero fraction (infinity)."""
    ne, nm, bias = fmt
    q, kept, rem, half, dn = _split(torch.where(m == 0, torch.ones_like(m), m), e, fmt)
    kept = kept + ((dn > 0) & ((rem > half) | ((rem == half) & ((kept & 1) == 1)))).to(torch.int64)
    inf = ((1 << ne) - 1) << nm
    mag = torch.where(m == 0, torch.zeros_like(m), (torch.clamp(q + bias + nm - 1, min=0) << nm) + kept)
    return (sign << (ne + nm)) | torch.clamp(mag, max=inf)


def _e4m3(sign, m, e):
    """E4M3 of (-1)^sign * m * 2^e (exact, 0 <= m < 2^61): round to nearest even, saturate at 448."""
    mag = _round(torch.zeros_like(sign), m, e, E4M3_WIDE)
    return (sign << 7) | torch.clamp(mag, max=E4M3_MAX)


def _f32_decode(bits):
    return _decode(bits, F32)


def _f32(sign, m, e, inf, nan):
    """F32 bits of one rounding of (-1)^sign * m * 2^e; inf and NaN as given (a NaN is F32_NAN)."""
    b = _round(sign, torch.where(inf | nan, torch.zeros_like(m), m), e, F32_FMT)
    b = torch.where(inf, (sign << 31) | F32_INF, b)
    return torch.where(nan, torch.full_like(b, F32_NAN), b)


def f32_mul(x_bits, y_bits):
    """RN(x * y) of two F32 patterns: the bits of FMUL without FTZ (a NaN product is F32_NAN)."""
    xs, xm, xe, xi, xn = _f32_decode(x_bits)
    ys, ym, ye, yi, yn = _f32_decode(y_bits)
    nan = xn | yn | (xi & (ym == 0) & ~yi) | (yi & (xm == 0) & ~xi)
    return _f32(xs ^ ys, xm * ym, xe + ye, (xi | yi) & ~nan, nan)


def f32_div(n_bits, d_bits):
    """RN(n / d) of two F32 patterns (IEEE division, subnormal results kept): the quotient's significand is an integer
    division with 27+ bits and a sticky bit below them, which no tie of a 24-bit result can fall between."""
    ns, nm, ne, ni, nn = _f32_decode(n_bits)
    ds, dm, de, di, dn = _f32_decode(d_bits)
    nan = nn | dn | (ni & di) | ((nm == 0) & ~ni & (dm == 0) & ~di)
    inf = (ni | ((dm == 0) & ~di)) & ~nan
    zero = (nm == 0) & ~ni | di
    num = torch.where(zero | inf | nan, torch.zeros_like(nm), nm) << 36  # nm < 2^24: quotient > 2^36 / 2^24
    den = torch.where(dm == 0, torch.ones_like(dm), dm)
    q = num // den
    sticky = ((num - q * den) != 0).to(torch.int64)
    b = _round(ns ^ ds, (q << 1) | sticky, ne - de - 37, F32_FMT)
    b = torch.where(inf, ((ns ^ ds) << 31) | F32_INF, b)
    return torch.where(nan, torch.full_like(b, F32_NAN), b)


def _const(v):
    return torch.tensor([v], dtype=torch.int64)


ONE, F448 = 0x3F800000, 0x43E00000
INV_448 = int(f32_div(_const(ONE), _const(F448))[0])  # RN(1 / 448) = 0x3B124925


def _flush(bits):
    """An F32 subnormal flushed to a zero of its sign (what .ftz does to an operand or result)."""
    return torch.where((bits & 0x7F800000) == 0, bits & 0x80000000, bits)


def reference_multiplier(a_bits):
    """m = RN(RN(1 / a) * 448) of clamped amax patterns a (int64, any device): RN(1 / a) is an F32 subnormal for
    a > 2^126 and is kept."""
    return f32_mul(f32_div(torch.full_like(a_bits, ONE), a_bits), torch.full_like(a_bits, F448))


def _widen_abs(bits, src):
    """|x| of src patterns (int64, low bits) as F32 bits, as the amax kernel widens them: F32 as it is, BF16 by a
    shift (sNaN payloads kept), F16 exactly, its NaNs as F32_NAN."""
    if src == F32:
        return bits & 0x7FFFFFFF
    if src == BF16:
        return (bits & 0x7FFF) << 16
    w = reference_cast(bits & 0x7FFF, F16, F32)
    return torch.where(w == NAN, torch.full_like(w, F32_NAN), w)


def widen(bits, src):
    """x of src patterns as F32 bits (signed; an F16 NaN as F32_NAN, a BF16 pattern shifted)."""
    sign = (bits >> (31 if src == F32 else 15)) & 1
    w = _widen_abs(bits, src)
    return torch.where(w == F32_NAN, w, w | (sign << 31))


def reference_block_scales(bits, src, R, C, block):
    """(a_bits, s_bits), int64 tensors of ceil(R / br) x ceil(C / bc), of the R x C weight whose src patterns are
    ``bits`` (row-major, any integer tensor, any device); ``None`` in block is the whole dimension."""
    br, bc = min(block[0] or R, R), min(block[1] or C, C)
    gR, gC = -(-R // br), -(-C // bc)
    w = _widen_abs(bits.to(torch.int64).reshape(R, C), src)
    padded = torch.zeros(gR * br, gC * bc, dtype=torch.int64, device=w.device)
    padded[:R, :C] = w
    top = padded.view(gR, br, gC, bc).amax(dim=(1, 3))
    a = torch.where(top > F32_INF, top, torch.clamp(top, min=FLOOR))
    return a, f32_mul(a, torch.full_like(a, INV_448))


def reference_quant(x_bits, src, m_bits):
    """E4M3 codes (int64) of src elements x (patterns ``x_bits``) times multipliers m (F32 patterns of one shape)."""
    xs, xm, xe, xi, xn = _decode(x_bits, src)
    ms, mm, me, mi, mn = _f32_decode(m_bits)
    nan = xn | mn | (xi & (mm == 0) & ~mi) | (mi & (xm == 0) & ~xi)
    inf = (xi | mi) & ~nan
    sign = xs ^ ms
    f = _f32(sign, torch.where(inf | nan, torch.zeros_like(xm), xm * mm), xe + me, inf, nan)
    fs, fm, fe, fi, _ = _f32_decode(f)
    q = _e4m3(fs, fm, fe)
    q = torch.where(fi, (fs << 7) | E4M3_MAX, q)
    return torch.where(nan, torch.full_like(q, E4M3_NAN), q)


def quant_one_rounding(x_bits, src, m_bits):
    """What a kernel that rounded the exact product once, straight to E4M3, would give."""
    xs, xm, xe, xi, xn = _decode(x_bits, src)
    ms, mm, me, mi, mn = _f32_decode(m_bits)
    nan = xn | mn | (xi & (mm == 0) & ~mi) | (mi & (xm == 0) & ~xi)
    inf = (xi | mi) & ~nan
    sign = xs ^ ms
    q = _e4m3(sign, torch.where(inf | nan, torch.zeros_like(xm), xm * mm), xe + me)
    q = torch.where(inf, (sign << 7) | E4M3_MAX, q)
    return torch.where(nan, torch.full_like(q, E4M3_NAN), q)


def wrong_multipliers(a_bits):
    """The multipliers of four wrong forms: one rounding of 448 / a; RN(1 / s); and RN(1 / a) flushed to zero (the
    ``.ftz`` reciprocal)."""
    s = f32_mul(a_bits, torch.full_like(a_bits, INV_448))
    return {
        "one rounding, RN(448 / a)": f32_div(torch.full_like(a_bits, F448), a_bits),
        "from s, RN(1 / s)": f32_div(torch.full_like(a_bits, ONE), s),
        "flush-to-zero reciprocal": f32_mul(_flush(f32_div(torch.full_like(a_bits, ONE), a_bits)),
                                            torch.full_like(a_bits, F448)),
    }


# --------------------------------------------------------------------------------------------- the value sets


def _f32_bits(x) -> int:
    with np.errstate(over="ignore"):  # past FLT_MAX: infinity, which no a admits
        return int(np.array(x, np.float32).view(np.uint32))


def _search(pred, n, seed):
    """n F32 patterns a (clamped-amax range: 2^-13 .. 2^127) with pred(a, m) true somewhere, from seeded draws."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randint(0x39000000, 0x7F000000, (1 << 14,), generator=g, dtype=torch.int64)
    hit = a[pred(a, reference_multiplier(a))]
    assert hit.numel() >= n
    return hit[:n].tolist()


def structured_amax():
    if not _STRUCTURED:
        _STRUCTURED.extend(_structured_amax())
    return list(_STRUCTURED)


_STRUCTURED = []


def _structured_amax():
    """Clamped amax patterns where the multiplier goes wrong: a where m differs from RN(448 / a) and a where it differs
    from RN(1 / s); the floor and one F32 ulp either side of it; powers of two; 448, 65504 and earlier test values;
    values in (2^126, FLT_MAX], whose reciprocal is an F32 subnormal; infinity and NaNs."""
    one = _search(lambda a, m: m != wrong_multipliers(a)["one rounding, RN(448 / a)"], 12, 1)
    from_s = _search(lambda a, m: m != wrong_multipliers(a)["from s, RN(1 / s)"], 12, 2)
    pow2 = [(127 + k) << 23 for k in (-13, -12, -7, -1, 0, 1, 3, 9, 15, 16, 40, 100, 126, 127)]
    top = [0x7E800001, 0x7EC00000, 0x7F000001, 0x7F400000, 0x7F7FFFFE, FLT_MAX]
    fixed = [FLOOR - 1, FLOOR, FLOOR + 1, F448, 0x477FE000] + [_f32_bits(v) for v in (3.0, 0.013, 1000.0, 1e30, 0.1)]
    return sorted(set(one + from_s + pow2 + top + fixed)) + [F32_INF, 0x7FC00000, 0x7F800001]


def raw_amax_edges():
    """Block maxima (|x| bits) that the floor clamps: 0, subnormals, floor - 1 ulp."""
    return [0, 1, 0x00400000, 0x007FFFFF, 0x00800000, FLOOR - 1]


def e4m3_values():
    """Every finite non-negative E4M3 value as an exact Fraction, ascending."""
    out = [Fraction(k, 1 << 9) for k in range(8)]
    for e in range(-6, 9):
        out += [Fraction(8 + f, 8) * Fraction(2) ** e for f in range(8 if e < 8 else 7)]
    return out


def product_targets():
    """F32 values that RN(x * m) should land on: every E4M3 tie (normal and subnormal), 448 and 464 - 1 ulp, and their
    F32 neighbours; as F32 patterns."""
    v = e4m3_values()
    ties = [(lo + hi) / 2 for lo, hi in zip(v, v[1:])] + [Fraction(464)]
    out = set()
    for t in ties + [Fraction(448)]:
        b = _f32_bits(float(t))
        assert Fraction(float(t)) == t
        out.update((b - 1, b, b + 1))
    out.update((0x43E7FFFF, 0x43E7FFFE))  # 464 - 1 and 2 ulps
    return sorted(out)


def solved_f32(a_bits):
    """For one finite clamped amax a: x patterns (both signs, |x| <= a) that make RN(x * m) land on the product
    targets, from the F32 nearest to target / m and 2 ulps either side of it; and x = +-a."""
    m = int(reference_multiplier(_const(a_bits))[0])
    mv = _fraction_value(m, F32)[1]
    xs = {a_bits}
    for t in product_targets():
        x0 = _f32_bits(float(_fraction_value(t, F32)[1] / mv))
        for d in range(-2, 3):
            x = x0 + d
            if 0 <= x <= a_bits:
                xs.add(x)
    pos = np.array(sorted(xs), np.int64)
    return np.concatenate([pos, pos | (1 << 31)])


def structured_f32_pairs():
    """(x_bits, a_bits): every finite structured a with its solved x values, as int64 tensors."""
    xs, as_ = [], []
    for a in structured_amax():
        if a >= F32_INF:
            continue
        x = solved_f32(a)
        xs.append(x)
        as_.append(np.full(x.size, a, np.int64))
    return torch.from_numpy(np.concatenate(xs)), torch.from_numpy(np.concatenate(as_))


def random_f32_rows(n, seed, width=64, device="cpu"):
    """(x_bits, a_bits) of n random F32 patterns in rows of ``width``, a = each row's reference amax (NaN rows give
    their NaN, whose m is a NaN)."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randint(0, 1 << 32, (n,), dtype=torch.int64, device=device, generator=g)
    a, _ = reference_block_scales(x, F32, n // width, width, (1, None))
    return x, a.reshape(-1).repeat_interleave(width)


def sixteen_bit_pairs(src, device="cpu"):
    """(x_bits, a_bits): for every structured a, every src pattern with |x| <= a (every pattern under a NaN a, every
    non-NaN one under infinity)."""
    every = torch.arange(1 << 16, dtype=torch.int64, device=device)
    mag = _widen_abs(every, src)
    xs, as_ = [], []
    for a in structured_amax():
        keep = torch.ones_like(every, dtype=torch.bool) if a > F32_INF else (mag <= a)
        xs.append(every[keep])
        as_.append(torch.full((int(keep.sum()),), a, dtype=torch.int64, device=device))
    return torch.cat(xs), torch.cat(as_)


# --------------------------------------------------------------------------------------------- a Fraction oracle


def _fraction_e4m3(sign, x):
    """E4M3 of the exact (-1)^sign * x (x >= 0 a Fraction), ties to even, saturating at 448."""
    if x == 0:
        return sign << 7
    e = x.numerator.bit_length() - x.denominator.bit_length()
    if Fraction(2) ** e > x:
        e -= 1
    q = max(e, -6) - 3
    n = x / Fraction(2) ** q
    k = n.numerator // n.denominator
    if n - k > Fraction(1, 2) or (n - k == Fraction(1, 2) and k % 2):
        k += 1
    if k >> 4:
        k, q = k >> 1, q + 1
    if k * Fraction(2) ** q >= 448:
        return (sign << 7) | E4M3_MAX
    field = q + 3 + 7 if k >> 3 else 0
    return (sign << 7) | (field << 3) | (k & 7)


def fraction_multiplier(a):
    _, av = _fraction_value(a, F32)
    if av == "nan":
        return "nan"
    if av == "inf":
        return 0
    r = _fraction_round(0, 1 / av, F32)
    return _fraction_round(0, _fraction_value(r, F32)[1] * 448, F32)


def fraction_quant(x, src, m):
    """reference_quant of one pair, with Python integers and Fractions only."""
    xs, xv = _fraction_value(x, src)
    ms, mv = _fraction_value(m, F32)
    if "nan" in (xv, mv) or (xv == "inf" and mv == 0) or (mv == "inf" and xv == 0):
        return E4M3_NAN
    if "inf" in (xv, mv):
        return ((xs ^ ms) << 7) | E4M3_MAX
    f = _fraction_round(xs ^ ms, xv * mv, F32)
    fs, fv = _fraction_value(f, F32)
    if fv == "inf":
        return (fs << 7) | E4M3_MAX
    return _fraction_e4m3(fs, fv)


# --------------------------------------------------------------------------------------------- the rounding classes


def _e4m3_tie(f_bits):
    """Whether the F32 patterns are finite, non-zero and exactly on a tie between two E4M3 values (or on 464)."""
    s, m, e, inf, nan = _f32_decode(f_bits)
    _, kept, rem, half, dn = _split(torch.where(m == 0, torch.ones_like(m), m), e, E4M3_WIDE)
    return ~inf & ~nan & (m != 0) & (dn >= 1) & (rem == half)


def classes(x_bits, src, a_bits):
    """Masks of the pairs in each class; P = RN(x * m) as F32, X the exact product."""
    m_bits = reference_multiplier(a_bits)
    p = f32_mul(widen(x_bits, src), m_bits)
    mag = p & 0x7FFFFFFF
    ps, pm, pe, pi, pn = _f32_decode(p)
    fin = ~pi & ~pn & (pm != 0)
    normal = mag >= 0x3C800000  # 2^-6, E4M3's smallest normal
    out = {}
    for name, rng in (("normal", normal), ("subnormal", ~normal)):
        out[f"P on an E4M3 tie, {name}"] = fin & rng & _e4m3_tie(p)
        out[f"P 1 ulp below an E4M3 tie, {name}"] = fin & rng & _e4m3_tie(p + 1)
        out[f"P 1 ulp above an E4M3 tie, {name}"] = fin & rng & _e4m3_tie(p - 1)
    ref = reference_quant(x_bits, src, m_bits)
    out["double rounding: X off a tie that P lands on, one rounding differs"] = \
        fin & _e4m3_tie(p) & (ref != quant_one_rounding(x_bits, src, m_bits))
    out["top: 448 <= |P| < 464"] = fin & (mag >= F448) & (mag < 0x43E80000)
    out["x = a"] = (x_bits & 0xFFFFFFFF) == a_bits
    out["bottom: P = +2^-10"] = p == 0x3A800000
    out["bottom: P = -2^-10"] = p == 0xBA800000
    out["a > 2^126: RN(1 / a) subnormal"] = (a_bits > 0x7E800000) & (a_bits < F32_INF) & fin
    return out


# --------------------------------------------------------------------------------------------- the tests


def _model():
    from tests.test_device_file_fp8_cpu import model_amax, model_q, model_scale

    return model_amax, model_scale, model_q


def _as_float(bits, t):
    w = 8 * t.itemsize
    b = bits & ((1 << w) - 1)
    signed = torch.where(b >= 1 << (w - 1), b - (1 << w), b)
    return signed.to({4: torch.int32, 2: torch.int16}[t.itemsize]).view(t)


def _check_q_against_model(x_bits, src, a_bits, what):
    """reference_quant against the torch CPU model of one element per row: bits where the model gives no NaN and the
    product stays below 464 (c10 gives NaN from there on, the kernel saturates), NaN where the model gives NaN."""
    _, _, model_q = _model()
    for lo in range(0, x_bits.numel(), 1 << 20):
        xb, ab = x_bits[lo : lo + (1 << 20)], a_bits[lo : lo + (1 << 20)]
        ref = reference_quant(xb, src, reference_multiplier(ab))
        got = model_q(_as_float(xb, src)[:, None], _as_float(ab, F32)[:, None], (1, 1)).view(torch.uint8)
        got = got.reshape(-1).to(torch.int64)
        nan = (got & 0x7F) == 0x7F
        p = f32_mul(widen(xb, src), reference_multiplier(ab))
        sat = ((p & 0x7FFFFFFF) >= 0x43E80000) & ((p & 0x7FFFFFFF) <= F32_INF)
        assert not sat.any() or src == F32, what
        bad = (~nan & ~sat & (ref != got)).nonzero().flatten()[:6]
        assert not bad.numel(), (what, [(hex(int(xb[k])), hex(int(ab[k])), hex(int(ref[k])), hex(int(got[k])))
                                        for k in bad])
        assert torch.equal(nan & ~sat, (ref == E4M3_NAN) & ~sat), what


def test_every_16_bit_pattern_under_every_structured_amax_equals_the_torch_cpu_model():
    for src in (F16, BF16):
        x, a = sixteen_bit_pairs(src)
        _check_q_against_model(x, src, a, ("every pattern", src))


def test_structured_and_random_f32_sets_equal_the_torch_cpu_model():
    x, a = structured_f32_pairs()
    _check_q_against_model(x, F32, a, "structured F32")
    x, a = random_f32_rows(1 << 20, seed=7)
    _check_q_against_model(x, F32, a, "random F32")


def test_block_scales_equal_the_torch_cpu_model():
    """a and s of weights with NaN payloads, infinities, zeros, subnormals, the floor and its neighbours, against
    model_amax / model_scale; a NaN a or s must be a NaN there (the CPU keeps payloads, the device makes F32_NAN)."""
    model_amax, model_scale, _ = _model()
    g = torch.Generator().manual_seed(3)
    for src in (F32, F16, BF16):
        bits = torch.randint(0, 1 << (8 * src.itemsize), (97, 131), generator=g, dtype=torch.int64)
        special = torch.tensor(raw_amax_edges() + [FLOOR + 1, F32_INF], dtype=torch.int64)
        if src != F32:  # zero, subnormals, the smallest normal and infinity of the 16-bit type
            special = torch.tensor([0, 1, 0x3FF, 0x7C00 if src == F16 else 0x7F80, 0x0400], dtype=torch.int64)
        bits[::7, ::5] = special[torch.arange(bits[::7, ::5].numel()) % special.numel()].view(bits[::7, ::5].shape)
        small = torch.randint(0, 1 << 8, (97, 131), generator=g) | (0x3000 if src != F32 else 0x30000000)
        for block in ((8, 16), (1, None), (None, 1), (5, 7), (None, None)):
            for w_bits in (bits, small):
                a, s = reference_block_scales(w_bits, src, 97, 131, block)
                blk = (min(block[0] or 97, 97), min(block[1] or 131, 131))
                ma = model_amax(_as_float(w_bits, src), blk)
                ms = model_scale(ma)
                ma_b, ms_b = (v.view(torch.int32).to(torch.int64) & 0xFFFFFFFF for v in (ma, ms))
                nan = torch.isnan(ma)
                assert torch.equal(nan, a > F32_INF) and torch.equal(nan, s > F32_INF), (src, block)
                assert torch.equal(a[~nan], ma_b[~nan]) and torch.equal(s[~nan], ms_b[~nan]), (src, block)
                if src != F16:  # BF16 and F32 NaN payloads widen by a shift: the model keeps them too
                    assert torch.equal(a, ma_b), (src, block)
                assert (s[nan] == F32_NAN).all()


def test_reference_equals_a_fraction_rounding_on_sampled_pairs_of_every_class_and_past_448():
    x, a = structured_f32_pairs()
    masks = classes(x, F32, a)
    g = torch.Generator().manual_seed(5)
    picks = []
    for mk in masks.values():
        idx = mk.nonzero().flatten()
        picks.append(idx[torch.randperm(idx.numel(), generator=g)[:60]])
    picks = torch.cat(picks)
    xs, as_ = x[picks].tolist(), a[picks].tolist()
    rng = random.Random(9)
    for _ in range(300):  # x past a: the saturating region, F32 overflow and F32 subnormal products
        av = rng.choice(structured_amax())
        xs.append(rng.randrange(1 << 32))
        as_.append(av)
    xt, at = torch.tensor(xs), torch.tensor(as_)
    mt = reference_multiplier(at)
    ref = reference_quant(xt, F32, mt).tolist()
    for k, (xb, ab, mb) in enumerate(zip(xs, as_, mt.tolist())):
        fm = fraction_multiplier(ab)
        assert (fm == "nan" and mb == F32_NAN) or fm == mb, (hex(ab), hex(mb), fm)
        assert ref[k] == fraction_quant(xb, F32, mb), (hex(xb), hex(ab), hex(mb), hex(ref[k]))
    for src in (F16, BF16):  # 16-bit x times random multipliers, the satfinite region included
        xb = torch.randint(0, 1 << 16, (400,), generator=g, dtype=torch.int64)
        mb = torch.randint(0, 0x7F800000, (400,), generator=g, dtype=torch.int64)
        ref = reference_quant(xb, src, mb).tolist()
        for k, (x1, m1) in enumerate(zip(xb.tolist(), mb.tolist())):
            assert ref[k] == fraction_quant(x1, src, m1), (src, hex(x1), hex(m1), hex(ref[k]))


def test_reference_spot_values():
    """Values fixed by the formats themselves, written out so that the reference's arithmetic cannot drift."""

    def m_of(a):
        return int(reference_multiplier(_const(a))[0])

    def q_of(x, src, m):
        return int(reference_quant(_const(x), src, _const(m))[0])

    assert INV_448 == 0x3B124925 == _f32_bits(np.float32(1) / np.float32(448))
    assert m_of(F448) == ONE  # RN(RN(1 / 448) * 448) = 1
    assert m_of(0x3F800000) == F448
    # a = 3: RN(RN(1 / 3) * 448) = 0x43155556, while 448 / 3 rounded once is 0x43155555
    assert m_of(0x40400000) == 0x43155556
    assert int(wrong_multipliers(_const(0x40400000))["one rounding, RN(448 / a)"][0]) == 0x43155555
    assert m_of(F32_INF) == 0 and m_of(0x7FC00000) == F32_NAN
    # a = FLT_MAX: RN(1 / a) = 2^-128 (0x00200000, subnormal), m = 1.75 * 2^-120 = 0x03E00000
    assert int(f32_div(_const(ONE), _const(FLT_MAX))[0]) == 0x00200000 and m_of(FLT_MAX) == 0x03E00000
    assert int(wrong_multipliers(_const(FLT_MAX))["flush-to-zero reciprocal"][0]) == 0
    assert q_of(FLT_MAX, F32, 0x03E00000) == 0x7E  # x = a = FLT_MAX quantizes to 448
    assert q_of(0x3F800000, F32, ONE) == 0x38 and q_of(0xBF800000, F32, ONE) == 0xB8  # +-1
    assert q_of(0x43E00000, F32, ONE) == 0x7E and q_of(0x43E7FFFF, F32, ONE) == 0x7E  # 448, 464 - ulp
    assert q_of(0x43E80000, F32, ONE) == 0x7E and q_of(0x7F7FFFFF, F32, ONE) == 0x7E  # satfinite: 464, FLT_MAX
    assert q_of(0xC3F00000, F32, ONE) == 0xFE and q_of(0xFF800000, F32, ONE) == 0xFE  # -480, -inf
    assert q_of(0x7F800000, F32, 0) == E4M3_NAN and q_of(0xFFC00000, F32, ONE) == E4M3_NAN  # inf * 0, -NaN
    assert q_of(0x3A800000, F32, ONE) == 0x00 and q_of(0xBA800000, F32, ONE) == 0x80  # +-2^-10: the tie goes to 0
    assert q_of(0x3A800001, F32, ONE) == 0x01 and q_of(0x3B000000, F32, ONE) == 0x01  # just above it; 2^-9
    assert q_of(0x80000001, F32, ONE) == 0x80  # a negative tiny value keeps its sign
    assert q_of(0x3F880000, F32, ONE) == 0x38 and q_of(0x3F980000, F32, ONE) == 0x3A  # 1 + 1/16 even, 1 + 3/16 up
    # double rounding (a pair of the structured set, a = floor - 1 ulp): X lies just above the tie 1.0625 * 2^-6
    # between 2^-6 (0x08) and 1.125 * 2^-6 (0x09); F32 rounds X down onto the tie (0x3C880000), which goes to the even
    # code 0x08, while one rounding of X gives 0x09
    x, m = 0x317EA776, 0x4A88B801
    assert int(f32_mul(_const(x), _const(m))[0]) == 0x3C880000
    assert q_of(x, F32, m) == 0x08 and int(quant_one_rounding(_const(x), F32, _const(m))[0]) == 0x09
    assert q_of(0x7C01, F16, ONE) == E4M3_NAN and q_of(0x7F81, BF16, ONE) == E4M3_NAN
    assert q_of(0x0001, F16, 0x4B800000) == 0x38  # the smallest F16 subnormal, 2^-24, times 2^24
    a, s = reference_block_scales(torch.tensor([0x7F81, 0x3F80, 0xFFC1, 0]), BF16, 2, 2, (None, None))
    assert int(a) == 0x7FC10000 and int(s) == F32_NAN  # the largest |NaN| bits win, s is the canonical NaN
    a, s = reference_block_scales(torch.tensor([0x7C01, 0x3C00]), F16, 1, 2, (1, 2))
    assert int(a) == F32_NAN and int(s) == F32_NAN
    a, s = reference_block_scales(torch.tensor([0x0001, 0x8000]), F16, 1, 2, (1, 2))
    assert int(a) == FLOOR and int(s) == int(f32_mul(_const(FLOOR), _const(INV_448))[0])
    a, _ = reference_block_scales(torch.tensor([0x0001, 0x83FF]), F16, 1, 2, (1, 1))
    assert a.tolist() == [[FLOOR, FLOOR]]  # F16 subnormals widen to normal F32 values below the floor
    a, s = reference_block_scales(torch.tensor([F32_INF | (1 << 31), 0x7F800001]), F32, 1, 2, (1, 2))
    assert int(a) == 0x7F800001 and int(s) == F32_NAN  # NaN beats infinity, its sNaN payload kept


def test_the_sets_reach_every_class_and_every_wrong_form_gives_other_bits():
    """Counts per class on the structured F32 pairs, and on them plus the 16-bit sets the number of pairs where each
    wrong form of the arithmetic gives other codes than the reference."""
    x, a = structured_f32_pairs()
    masks = classes(x, F32, a)
    counts = {name: int(mk.sum()) for name, mk in masks.items()}
    for name, n in counts.items():
        assert n >= 20, f"{name}: {n} pairs in the structured F32 set ({x.numel()} pairs); all counts: {counts}"
    m = reference_multiplier(a)
    ref = reference_quant(x, F32, m)
    differ = {}
    for name, wm in wrong_multipliers(a).items():
        differ[name] = int((reference_quant(x, F32, wm) != ref).sum())
    differ["one rounding of the exact product to E4M3"] = int((quant_one_rounding(x, F32, m) != ref).sum())
    for src in (F16, BF16):
        xs, as_ = sixteen_bit_pairs(src)
        r16 = reference_quant(xs, src, reference_multiplier(as_))
        for name, wm in wrong_multipliers(as_).items():
            if src == F16 and name == "flush-to-zero reciprocal":
                continue  # under a > 2^126, every F16 value times m rounds to zero either way
            differ[f"{name}, {src}"] = int((reference_quant(xs, src, wm) != r16).sum())
    for name, n in differ.items():
        assert n >= 10, f"{name}: {n} pairs differ from the reference; all: {differ}"
