"""An integer-exact statement of the FP8 dequantization the scaled box copy performs, and the CPU tests that make it
trustworthy.

The contract (DESIGN §5.18) is two roundings: the FP8 element and its scale are decoded exactly, their exact product
is rounded once to F32 (round to nearest even, subnormals kept, overflow to infinity), and that F32 value is rounded
once more to the target type.  Rounding the exact product straight to a 16-bit target gives other bits for a few
products in a million; ``structured_f32_scales`` builds F32 scales that reach those products, and every other rounding
edge of the two steps, on purpose.

``reference_dequant`` uses int64 tensor arithmetic only -- no float type is formed -- so it is independent of the
``FMUL`` and ``cvt`` instructions that the kernel and torch's CUDA expression issue, and it runs unchanged on CPU and
CUDA tensors (tests/test_scaled_box_paths_gpu.py runs it on the device).  Note that "exact in float64, then ``.to(T)``"
is no independent reference: torch's CPU float64 -> bfloat16 goes through F32 too, so it double-rounds like the kernel.

It is checked three ways: against torch's CPU ``(w.float() * s.float()).to(T)`` for every FP8 pattern times every F16
and BF16 scale and times the structured and random F32 scales; against a plain ``fractions.Fraction`` rounding on
sampled pairs of every class; and by showing that the structured set holds pairs of every class, and that on its
double-rounding pairs a single rounding gives other bits."""
import math
import random
from fractions import Fraction

import numpy as np
import pytest
import torch

from tests.test_cast_reference_cpu import FORMATS, NAN, reference_cast

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
# (exponent bits, fraction bits, bias); E4M3 has no infinities and one NaN magnitude (S.1111.111), E5M2 is IEEE-like
FP8 = {E4M3: (4, 3, 7), E5M2: (5, 2, 15)}
TARGETS = [BF16, F16, F32]
INT_VIEW = {F32: torch.int32, F16: torch.int16, BF16: torch.int16, E4M3: torch.uint8, E5M2: torch.uint8}


def _decode(bits, t):
    """(sign, m, e, inf, nan) of the type-t patterns in the low bits of ``bits``: a finite value is m * 2^e exactly."""
    ne, nm, bias = FP8[t] if t in FP8 else FORMATS[t]
    x = bits.to(torch.int64) & ((1 << (1 + ne + nm)) - 1)
    sign = x >> (ne + nm)
    exp = (x >> nm) & ((1 << ne) - 1)
    frac = x & ((1 << nm) - 1)
    top = exp == (1 << ne) - 1
    if t == E4M3:
        inf, nan = torch.zeros_like(top), top & (frac == (1 << nm) - 1)
    else:
        inf, nan = top & (frac == 0), top & (frac != 0)
    normal = exp != 0
    m = torch.where(normal, frac | (1 << nm), frac)
    e = torch.where(normal, exp, torch.ones_like(exp)) - bias - nm
    return sign, m, e, inf, nan


def _log2(m):
    """floor(log2(m)) for 1 <= m < 2^32 (0 for m = 0)."""
    p = torch.zeros_like(m)
    for k in (16, 8, 4, 2, 1):
        p = torch.where((m >> (p + k)) != 0, p + k, p)
    return p


def _split(m, e, t):
    """Rounding m * 2^e (0 < m < 2^32) to type t: (q, kept, rem, half, dn).  2^q is t's quantum at the value (that of
    its binade, or of t's subnormal range), ``kept`` the value in quanta rounded toward zero, ``rem`` the dropped part
    in units of 2^e and ``half`` the tie in those units (0 when nothing is dropped), ``dn`` the count of dropped bits."""
    ne, nm, bias = FORMATS[t]
    q = torch.clamp(_log2(m) + e, min=1 - bias) - nm
    r = q - e
    dn = torch.clamp(r, 0, 62)  # m < 2^32: 62 bits drop everything and leave the tie bit above m
    kept = (m << torch.clamp(-r, min=0)) >> dn
    rem = m & ((torch.ones_like(m) << dn) - 1)
    half = torch.where(dn > 0, torch.ones_like(m) << torch.clamp(dn - 1, min=0), torch.zeros_like(m))
    return q, kept, rem, half, dn


def round_exact(sign, m, e, t):
    """The bits (int64) of type t nearest to (-1)^sign * m * 2^e (0 <= m < 2^32), ties to even, overflow to
    infinity: one rounding of an exact value."""
    ne, nm, bias = FORMATS[t]
    q, kept, rem, half, dn = _split(m, e, t)
    kept = kept + ((dn > 0) & ((rem > half) | ((rem == half) & ((kept & 1) == 1)))).to(torch.int64)
    # biased exponent - 1 in the exponent field plus a significand that still holds its leading bit (see
    # reference_cast): a rounding carry moves into the exponent, a subnormal's field is 0
    inf = ((1 << ne) - 1) << nm
    mag = torch.where(m == 0, torch.zeros_like(m), (torch.clamp(q + bias + nm - 1, min=0) << nm) + kept)
    return (sign << (ne + nm)) | torch.clamp(mag, max=inf)


def exact_product(w_bits, fmt, s_bits, stype):
    """The exact product of FP8 elements and scales: (sign, m, e, inf, nan), value (-1)^sign * m * 2^e (m < 2^28)
    where it is finite.  NaN: either factor a NaN, or 0 times infinity; infinity: an infinite factor otherwise."""
    ws, wm, we, winf, wnan = _decode(w_bits, fmt)
    ss, sm, se, sinf, snan = _decode(s_bits, stype)
    nan = wnan | snan | (winf & (sm == 0) & ~sinf) | (sinf & (wm == 0) & ~winf)
    inf = (winf | sinf) & ~nan
    return ws ^ ss, wm * sm, we + se, inf, nan


def _f32(sign, m, e, inf, nan):
    """The F32 bits of one rounding to F32; a NaN as 0x7FC00000, which reference_cast turns into its NAN marker."""
    b = round_exact(sign, torch.where(inf | nan, torch.zeros_like(m), m), e, F32)
    b = torch.where(inf, (sign << 31) | 0x7F800000, b)
    return torch.where(nan, torch.full_like(b, 0x7FC00000), b)


def reference_dequant(w_bits, fmt, s_bits, stype, dst):
    """The ``dst`` bit patterns (int64, zero-extended) of FP8 elements (type ``fmt``, patterns ``w_bits``) times
    their scales (type ``stype``, patterns ``s_bits``; both any integer tensors of one shape, on any device): the exact
    product rounded to nearest even F32 (subnormals down to 2^-149, overflow to infinity), then that F32 value rounded
    to ``dst`` by ``reference_cast``.  ``NAN`` where the product is a NaN."""
    return reference_cast(_f32(*exact_product(w_bits, fmt, s_bits, stype)), F32, dst)


def single_rounding(w_bits, fmt, s_bits, stype, dst):
    """What a kernel that rounded the exact product once, straight to ``dst``, would give (``NAN`` for NaNs)."""
    sign, m, e, inf, nan = exact_product(w_bits, fmt, s_bits, stype)
    b = round_exact(sign, torch.where(inf | nan, torch.zeros_like(m), m), e, dst)
    ne, nm, _ = FORMATS[dst]
    b = torch.where(inf, (sign << (ne + nm)) | (((1 << ne) - 1) << nm), b)
    return torch.where(nan, torch.full_like(b, NAN), b)


# --------------------------------------------------------------------------------------------- the value sets


def _fp8_significands(fmt):
    """Every FP8 significand m8 of the format with the exponents e8 it takes (value m8 * 2^e8): subnormal significands
    only at the smallest exponent, normal ones at every finite exponent."""
    ne, nm, bias = FP8[fmt]
    emin = 1 - bias - nm
    emax = (1 << ne) - 1 - bias - nm - (1 if fmt == E5M2 else 0)
    top = (1 << (nm + 1)) - 1  # E4M3's largest significand at its largest exponent is its NaN
    return {m8: (emin, (emax - (fmt == E4M3 and m8 == top)) if m8 >> nm else emin) for m8 in range(1, top + 1)}


def _f32_pattern(ms, es):
    """The F32 bits of ms * 2^es, or None if that is no F32 value."""
    x = math.ldexp(ms, es)
    if not 0 < x < 2.0**128:
        return None
    b = int(np.array(x, np.float64).astype(np.float32).view(np.uint32))
    return b if float(np.uint32(b).view(np.float32)) == x else None


def _solve(m8, pattern, k0, tries=64):
    """ms = N / m8 for the first N = pattern(k), k = k0, k0 + 1, ..., that is a multiple of m8 with N / m8 < 2^24."""
    for k in range(k0, k0 + tries):
        n = pattern(k)
        if n is not None and n > 0 and n % m8 == 0 and n // m8 < 1 << 24:
            return n // m8
    return None


def _templates(fmt):
    """For each FP8 significand m8: (m8, ms, E) with the exact product m8 * ms * 2^E where a rounding class wants
    it."""
    e8min = min(lo for lo, _ in _fp8_significands(fmt).values())
    out = []
    rng = random.Random(FP8[fmt][1])  # seeded per format: where the searches for N start
    for m8 in _fp8_significands(fmt):
        # F32 ties in the normal range: N = K * 2^d + 2^(d - 1) (+-1) has 24 + d bits, d of them dropped
        for d in range(1, 5):
            for o in (-1, 0, 1):
                for k0 in ((1 << 23) + rng.randrange(1 << 22), (1 << 24) - 64 - rng.randrange(1 << 20)):
                    ms = _solve(m8, lambda k: (k << d) + (1 << (d - 1)) + o, k0)
                    if ms:
                        out.append((m8, ms, -(24 + d)))
        # F32 ties in the subnormal range: the product N * 2^(-149 - r) (N < 2^(23 + r)) drops r bits
        for r in range(1, -e8min + 1):
            for o in (-1, 0, 1):
                n0 = min(m8 << 23, 1 << (22 + r)) + rng.randrange(1 << 20)
                ms = _solve(m8, lambda k: ((k << r) + (1 << (r - 1)) + o) if ((k + 1) << r) <= 1 << (23 + r) else None,
                            n0 >> r)
                if ms:
                    out.append((m8, ms, -149 - r))
        # an F32 result exactly on a tie of a 16-bit target (h of its 24 significand bits dropped), reached from the
        # exact product on the odd side of that tie: N = Fsig * 2^d +- t, 0 < t <= 2^(d - 1)
        for h in (16, 13):
            for d in range(1, 5):
                for t in range(1, (1 << (d - 1)) + 1):
                    def pattern(b):
                        fsig = (b << h) | (1 << (h - 1))
                        return (fsig << d) + t if b % 2 == 0 else (fsig << d) - t
                    for b0 in ((1 << (23 - h)) + rng.randrange(1 << (22 - h)), (1 << (24 - h)) - 20):
                        ms = _solve(m8, pattern, b0, tries=20)
                        if ms:
                            out.append((m8, ms, -(23 + d)))
        # integers N near the edges: F16's largest values and its overflow tie, its subnormal bottom, F32's
        # normal bottom and overflow
        for x in (65504, 65520, 65536, 2.0**-24, 2.0**-25, 3 * 2.0**-26, 2.0**-14, 2.0**-126,
                  2.0**128 - 2.0**104, 2.0**128 - 2.0**103, 2.0**128):
            big_e = math.frexp(x)[1] - 23 - m8.bit_length()  # N / m8 between 2^22 and 2^24
            n = Fraction(x) / Fraction(2) ** big_e
            base = int(n / m8)
            for j in range(-3, 4):
                if 0 < base + j < 1 << 24:
                    out.append((m8, base + j, big_e))
    return out


def structured_f32_scales() -> np.ndarray:
    """F32 scale patterns (uint32, both signs) whose exact products with FP8 elements land where the two roundings
    go wrong: for every FP8 significand m8 of both formats, scales ms = N / m8 with integers N at and one unit either
    side of F32 ties in the normal and subnormal result ranges, at F32 results that are exactly BF16 or F16 ties
    reached from the odd side (where one rounding differs from two), and around F16's 65504 / 65520 edge, its subnormal
    bottom, F32's smallest normal and F32 overflow.  Each (ms, E) becomes a scale by the FP8 exponent that puts it
    nearest 1, so paired with every FP8 pattern a scale meets its significand at every exponent."""
    pats = set()
    for fmt in FP8:
        sig = _fp8_significands(fmt)
        for m8, ms, big_e in _templates(fmt):
            # the element m8 * 2^e8 and the scale ms * 2^(E - e8) have the product the class wants: take the e8 that
            # m8 has which makes the scale a finite F32 nearest 1
            lo, hi = sig[m8]
            for e8 in sorted(range(lo, hi + 1), key=lambda e8: abs(big_e - e8 + 23)):
                b = _f32_pattern(ms, big_e - e8)
                if b is not None:
                    pats.add(b)
                    break
    pos = np.array(sorted(pats), np.uint32)
    return np.concatenate([pos, pos | np.uint32(0x80000000)])


def random_f32_scales(n=1 << 16, seed=811) -> np.ndarray:
    """n random F32 patterns (uint32): every sign, exponent, NaN and infinity alike."""
    return np.random.default_rng(seed).integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)


def pairs(scales):
    """Every FP8 pattern times every scale: (w_bits, s_bits), int64, pattern-major within each scale."""
    s = torch.as_tensor(np.asarray(scales).astype(np.int64))
    return torch.arange(256, dtype=torch.int64).repeat(s.numel()), s.repeat_interleave(256)


# --------------------------------------------------------------------------------------------- the rounding classes


def _cmp(m, e, c):
    """The sign of m * 2^e - c (m < 2^28, c > 0 a constant with a significand below 2^26), exactly."""
    f = Fraction(c)
    ce = 0
    while f.denominator != 1:
        f, ce = f * 2, ce - 1
    cm = int(f)
    while cm % 2 == 0:
        cm, ce = cm // 2, ce + 1
    d = e - ce
    a = torch.where(d >= 0, m << torch.clamp(d, 0, 34), m)
    b = torch.where(d < 0, cm << torch.clamp(-d, 0, 36), torch.full_like(m, cm))
    return torch.sign(a - b)


def classes(w_bits, fmt, s_bits, stype=F32):
    """Masks of the pairs in each rounding class (finite non-zero exact products x, F = x rounded to F32)."""
    sign, m, e, inf, nan = exact_product(w_bits, fmt, s_bits, stype)
    fin = ~inf & ~nan & (m != 0)
    m = torch.where(fin, m, torch.ones_like(m))
    q, kept, rem, half, dn = _split(m, e, F32)
    normal = _cmp(m, e, 2.0**-126) >= 0
    out = {}
    for rng, where in (("normal", normal & (_cmp(m, e, 2.0**128) < 0)), ("subnormal", ~normal)):
        out[f"F32 tie, {rng}"] = fin & where & (dn >= 1) & (rem == half)
        out[f"F32 tie - 1, {rng}"] = fin & where & (dn >= 2) & (rem == half - 1)
        out[f"F32 tie + 1, {rng}"] = fin & where & (dn >= 2) & (rem == half + 1)
    # F lies exactly on a tie of t, and x on the side of it away from t's even neighbour: two roundings go to even,
    # one goes toward x
    f = _f32(sign, m, e, inf, nan)
    fs, fm, fe, finf, _ = _decode(f, F32)
    above = (rem != 0) & ((rem < half) | ((rem == half) & ((kept & 1) == 0)))  # F32 rounded x down
    for name, t, top in (("BF16", BF16, 2.0**128), ("F16", F16, 2.0**16)):  # (at and past `top` both give inf)
        _, tk, trem, thalf, tdn = _split(torch.where(fm == 0, torch.ones_like(fm), fm), fe, t)
        on_tie = fin & ~finf & (fm != 0) & (tdn >= 1) & (trem == thalf) & (rem != 0) & (_cmp(m, e, top) < 0)
        out[f"double rounding onto a {name} tie"] = on_tie & (above == ((tk & 1) == 0))
    between = lambda lo, hi: fin & (_cmp(m, e, lo) > 0) & (_cmp(m, e, hi) < 0)  # noqa: E731
    out["F16: 65504 < |x| < 65520"] = between(65504, 65520)
    out["F16: |x| = 65520"] = fin & (_cmp(m, e, 65520) == 0)
    out["F16: 65520 < |x| < 65536"] = between(65520, 65536)
    out["F16: 0 < |x| < 2^-25"] = fin & (_cmp(m, e, 2.0**-25) < 0)
    out["F16: |x| = 2^-25"] = fin & (_cmp(m, e, 2.0**-25) == 0)
    out["F16: 2^-25 < |x| < 2^-24"] = between(2.0**-25, 2.0**-24)
    # no FP8 x F32 product lies in (max + ulp / 2, 2^128): its significand would need more factors than 4 + 24 bits
    # give; E5M2's none in (max, max + ulp / 2) either, so the lower class starts at max itself
    out["F32: max <= |x| < max + ulp / 2"] = fin & (_cmp(m, e, 2.0**128 - 2.0**104) >= 0) & \
        (_cmp(m, e, 2.0**128 - 2.0**103) < 0)
    out["F32 overflow: 2^128 <= |x| < 2^129"] = fin & (_cmp(m, e, 2.0**128) >= 0) & (_cmp(m, e, 2.0**129) < 0)
    return out


# --------------------------------------------------------------------------------------------- a Fraction oracle


def _fraction_value(bits, fmt):
    """(sign, Fraction | 'inf' | 'nan') of one pattern, decoded by the format's definition."""
    ne, nm, bias = FP8[fmt] if fmt in FP8 else FORMATS[fmt]
    sign, exp, frac = bits >> (ne + nm) & 1, (bits >> nm) & ((1 << ne) - 1), bits & ((1 << nm) - 1)
    if exp == (1 << ne) - 1:
        if fmt == E4M3:
            if frac == (1 << nm) - 1:
                return sign, "nan"
        else:
            return sign, "nan" if frac else "inf"
    if exp == 0:
        return sign, Fraction(frac) * Fraction(2) ** (1 - bias - nm)
    return sign, Fraction(frac + (1 << nm)) * Fraction(2) ** (exp - bias - nm)


def _fraction_round(sign, x, t):
    """The bits of type t nearest to the exact (-1)^sign * x (x >= 0 a Fraction), ties to even."""
    ne, nm, bias = FORMATS[t]
    if x == 0:
        return sign << (ne + nm)
    big_e = x.numerator.bit_length() - x.denominator.bit_length()
    if Fraction(2) ** big_e > x:
        big_e -= 1
    q = max(big_e, 1 - bias) - nm
    n = x / Fraction(2) ** q
    k = n.numerator // n.denominator
    if n - k > Fraction(1, 2) or (n - k == Fraction(1, 2) and k % 2):
        k += 1
    if k >> (nm + 1):  # the carry into the next binade
        k, q = k >> 1, q + 1
    field = q + nm + bias if k >> nm else 0
    if field >= (1 << ne) - 1:
        return (sign << (ne + nm)) | (((1 << ne) - 1) << nm)
    return (sign << (ne + nm)) | (field << nm) | (k & ((1 << nm) - 1))


def fraction_dequant(w, fmt, s, stype, dst):
    """reference_dequant of one pair, with Python integers and Fractions only."""
    ws, wv = _fraction_value(w, fmt)
    ss, sv = _fraction_value(s, stype)
    sign = ws ^ ss
    if "nan" in (wv, sv) or (wv == "inf" and sv == 0) or (sv == "inf" and wv == 0):
        return NAN
    if "inf" in (wv, sv):
        f = (sign << 31) | 0x7F800000
    else:
        f = _fraction_round(sign, wv * sv, F32)
    fs, fv = _fraction_value(f, F32)
    if fv == "inf":
        de, dm, _ = FORMATS[dst]
        return (fs << (de + dm)) | (((1 << de) - 1) << dm)
    return _fraction_round(fs, fv, dst)


# --------------------------------------------------------------------------------------------- the tests


def _torch_bits(w_bits, fmt, s_bits, stype, dst):
    """torch's CPU (w.float() * s.float()).to(dst), as zero-extended bits, and its NaN mask."""
    w = w_bits.to(torch.uint8).view(fmt)
    s = (s_bits.to(torch.int64) & ((1 << (8 * stype.itemsize)) - 1))
    s = torch.where(s >= 1 << (8 * stype.itemsize - 1), s - (1 << (8 * stype.itemsize)), s).to(INT_VIEW[stype])
    y = (w.float() * s.view(stype).float()).to(dst)
    return y.view(INT_VIEW[dst]).to(torch.int64) & ((1 << (8 * dst.itemsize)) - 1), y.isnan()


def _check_against_torch(w_bits, fmt, s_bits, stype, what):
    for dst in TARGETS:
        ref = reference_dequant(w_bits, fmt, s_bits, stype, dst)
        want, nan = _torch_bits(w_bits, fmt, s_bits, stype, dst)
        assert torch.equal(ref == NAN, nan), (what, fmt, dst, int(((ref == NAN) != nan).sum()))
        bad = torch.nonzero(~nan & (ref != want)).flatten()[:8]
        assert not bad.numel(), (what, fmt, dst, [(hex(int(w_bits[k])), hex(int(s_bits[k]) & 0xFFFFFFFF),
                                                   hex(int(ref[k])), hex(int(want[k]))) for k in bad])


FMT_IDS = ["e4m3", "e5m2"]


@pytest.mark.parametrize("fmt", [E4M3, E5M2], ids=FMT_IDS)
@pytest.mark.parametrize("stype", [F16, BF16], ids=["f16", "bf16"])
def test_every_fp8_pattern_times_every_16_bit_scale_equals_torch_cpu(fmt, stype):
    """256 x 65 536 pairs into all three targets.  Every product is exact in F32 here (at most 4 + 11 significand
    bits) except where it leaves F32's range, so this pins decoding, signs, specials, subnormals and overflow."""
    for lo in range(0, 1 << 16, 1 << 13):
        w, s = pairs(np.arange(lo, lo + (1 << 13)))
        _check_against_torch(w, fmt, s, stype, ("16-bit scales", lo))


@pytest.mark.parametrize("fmt", [E4M3, E5M2], ids=FMT_IDS)
def test_structured_and_random_f32_scales_equal_torch_cpu(fmt):
    scales = np.concatenate([structured_f32_scales(), random_f32_scales()])
    for lo in range(0, scales.size, 1 << 13):
        w, s = pairs(scales[lo : lo + (1 << 13)])
        _check_against_torch(w, fmt, s, F32, ("F32 scales", lo))


_classes = {}


def structured_classes(fmt):
    """(w, s, masks) of every FP8 pattern times the structured F32 scales."""
    if fmt not in _classes:
        w, s = pairs(structured_f32_scales())
        _classes[fmt] = (w, s, classes(w, fmt, s))
    return _classes[fmt]


@pytest.mark.parametrize("dst", TARGETS, ids=["bf16", "f16", "f32"])
@pytest.mark.parametrize("fmt", [E4M3, E5M2], ids=FMT_IDS)
def test_the_structured_set_reaches_every_rounding_class(fmt, dst):
    """At least one pair of every class; on the double-rounding pairs of dst's own class, rounding the exact product
    once to dst gives other bits than the reference, so a kernel that rounds once fails on them."""
    w, s, masks = structured_classes(fmt)
    counts = {name: int(mk.sum()) for name, mk in masks.items()}
    for name, n in counts.items():
        assert n >= 1, f"{name}: {n} pairs of {FMT_IDS[fmt == E5M2]} x the structured set into {dst}"
    if dst != F32:
        mk = masks[f"double rounding onto a {'BF16' if dst == BF16 else 'F16'} tie"]
        ref = reference_dequant(w[mk], fmt, s[mk], F32, dst)
        one = single_rounding(w[mk], fmt, s[mk], F32, dst)
        same = int((ref == one).sum())
        assert same == 0, f"{same} of {int(mk.sum())} double-rounding pairs round alike once and twice"


@pytest.mark.parametrize("fmt", [E4M3, E5M2], ids=FMT_IDS)
def test_reference_equals_a_fraction_rounding_on_sampled_pairs_of_every_class(fmt):
    w, s, masks = structured_classes(fmt)
    g = torch.Generator().manual_seed(5)
    picks = []
    for mk in masks.values():
        idx = mk.nonzero().flatten()
        picks.append(idx[torch.randperm(idx.numel(), generator=g)[:150]])
    rw, rs = pairs(random_f32_scales()[:16])
    picks = torch.cat(picks)
    w_all, s_all = torch.cat([w[picks], rw]), torch.cat([s[picks], rs])
    assert w_all.numel() >= 2000
    for dst in TARGETS:
        ref = reference_dequant(w_all, fmt, s_all, F32, dst).tolist()
        for k, (a, b) in enumerate(zip(w_all.tolist(), s_all.tolist())):
            assert ref[k] == fraction_dequant(a, fmt, b, F32, dst), (hex(a), hex(b), dst, hex(ref[k]))


def test_reference_spot_values():
    """Values fixed by the formats themselves, written out so that the reference's arithmetic cannot drift."""

    def one(w, fmt, s, stype, dst, once=False):
        f = single_rounding if once else reference_dequant
        return int(f(torch.tensor([w]), fmt, torch.tensor([s]), stype, dst)[0])

    # 3 * 2^-9 * 0x3F865555: the exact product 0x192FFFF * 2^-32 rounds to F32 0x3BC98000 (a tie, to even), which is
    # a BF16 tie: two roundings give 0x3BCA (0.00616455078125), one gives 0x3BC9 (0.006134033203125)
    assert one(0x03, E4M3, 0x3F865555, F32, F32) == 0x3BC98000
    assert one(0x03, E4M3, 0x3F865555, F32, BF16) == 0x3BCA
    assert one(0x03, E4M3, 0x3F865555, F32, BF16, once=True) == 0x3BC9
    assert one(0x7E, E4M3, 0x3F800000, F32, F32) == 0x43E00000  # 448, E4M3's largest
    assert one(0x7F, E4M3, 0x3F800000, F32, BF16) == NAN and one(0xFF, E4M3, 0x3F800000, F32, F16) == NAN
    assert one(0x7C, E5M2, 0x3F800000, F32, F16) == 0x7C00  # E5M2 infinity
    assert one(0xFC, E5M2, 0xBF800000, F32, BF16) == 0x7F80  # -inf * -1
    assert one(0x7C, E5M2, 0x00000000, F32, F32) == NAN  # inf * 0
    assert one(0x00, E4M3, 0x7F800000, F32, F32) == NAN  # 0 * inf
    assert one(0x80, E4M3, 0x3F800000, F32, F32) == 0x80000000  # -0 * 1
    assert one(0x01, E4M3, 0x00800000, F32, F32) == 0x00004000  # 2^-9 * 2^-126 = 2^-135, an F32 subnormal
    assert one(0x03, E4M3, 0x00000100, F32, F32) == 0x00000002  # 3 * 2^-150: a tie between 1 and 2 * 2^-149, even
    assert one(0x01, E4M3, 0x00000100, F32, F32) == 0x00000000  # 2^-150: the tie between 0 and 2^-149 goes to 0
    assert one(0x81, E4M3, 0x00000180, F32, F32) == 0x80000001  # -0.75 * 2^-149 rounds to -2^-149
    assert one(0x7E, E4M3, 0x7F7FFFFF, F32, F32) == 0x7F800000  # 448 * max: overflow
    assert one(0x3C, E4M3, 0x4780_0000, F32, F16) == 0x7C00  # 1.5 * 65536: F16 overflow
    assert one(0x38, E4M3, 0x477FF000, F32, F16) == 0x7C00  # 1 * 65520: the F16 tie goes to infinity
    assert one(0x38, E4M3, 0x33000000, F32, F16) == 0x0000  # 1 * 2^-25: the tie at F16's bottom goes to 0
    assert one(0x3C, E5M2, 0x0001, F16, F32) == 0x33800000  # 1 * 2^-24, an F16 subnormal scale, widened exactly
    assert one(0x38, E4M3, 0x0001, BF16, F32) == 0x00010000  # a BF16 subnormal scale
