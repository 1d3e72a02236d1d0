"""An integer-exact statement of the F32 / F16 / BF16 conversions the device copies perform, and the CPU tests that
make it trustworthy: every non-NaN 16-bit pattern of both 16-bit types through its three conversions against torch's
CPU ``.to()``, and a structured F32 set (every exponent with the mantissas at and around every rounding tie, every F16
subnormal boundary, the F16 overflow edge, signed zeros and infinities) plus 2^26 random F32 patterns against torch's
CPU ``.to()`` and numpy's ``astype(np.float16)``.

``reference_cast`` uses int64 tensor arithmetic only -- no float type is ever formed -- so it is independent of the
``cvt`` instructions the kernels and torch's CUDA casts issue, and it runs unchanged on CPU and CUDA tensors
(tests/test_cast_paths_gpu.py runs it on the device)."""
import numpy as np
import pytest
import torch

# (exponent bits, fraction bits, bias)
FORMATS = {torch.float32: (8, 23, 127), torch.float16: (5, 10, 15), torch.bfloat16: (8, 7, 127)}
INT_VIEW = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}
NAN = -1  # what reference_cast returns for a NaN input: the NaN bits (sign, payload) are the device's to choose


def reference_cast(bits: torch.Tensor, src: torch.dtype, dst: torch.dtype) -> torch.Tensor:
    """The ``dst`` bit patterns (int64, zero-extended) of the ``src`` elements whose bit patterns are ``bits`` (any
    integer tensor; the low bits of each value are the pattern, sign extension is ignored), converted with IEEE 754
    round to nearest, ties to even; ``NAN`` where an input is a NaN.

    A finite input is decoded to its exact value m * 2^E (m an integer below 2^24) and rounded once to ``dst``: the
    destination's quantum 2^q is that of the input's binade, or of its subnormal range when the value lies below the
    smallest normal (F16 subnormals reach 2^-24, F32 ones 2^-149, BF16 ones 2^-133).  A result that rounds to 2^(emax
    + 1) or above becomes infinity (F16: every |x| >= 65520).  Widening (F16 / BF16 -> F32) never drops a bit.  F16 <->
    BF16 is that one rounding of the exact source value, which is what widening exactly to F32 and rounding once to the
    other type gives: F32 holds every F16 and BF16 value exactly, so there is no double rounding."""
    se, sm, sbias = FORMATS[src]
    de, dm, dbias = FORMATS[dst]
    x = bits.to(torch.int64) & ((1 << (1 + se + sm)) - 1)
    sign = x >> (se + sm)
    exp = (x >> sm) & ((1 << se) - 1)
    frac = x & ((1 << sm) - 1)
    special = exp == (1 << se) - 1  # infinities and NaNs
    normal = exp != 0
    m = torch.where(normal, frac | (1 << sm), frac)
    e = torch.where(normal, exp, torch.ones_like(exp)) - sbias - sm  # value = m * 2^e
    # p = floor(log2(m)) for m >= 1 (m < 2^24)
    p = torch.zeros_like(m)
    for k in (16, 8, 4, 2, 1):
        p = torch.where((m >> (p + k)) != 0, p + k, p)
    q = torch.clamp(p + e, min=1 - dbias) - dm  # the destination quantum's exponent
    r = q - e  # bits to drop (<= 0: exact)
    up = torch.clamp(-r, min=0)
    dn = torch.clamp(r, 0, 62)  # m < 2^24: 62 bits drop everything and leave the tie bit above m, as any r > 24 does
    kept = (m << up) >> dn
    rem = m & ((torch.ones_like(m) << dn) - 1)
    half = torch.where(dn > 0, torch.ones_like(m) << torch.clamp(dn - 1, min=0), torch.zeros_like(m))
    round_up = (dn > 0) & ((rem > half) | ((rem == half) & ((kept & 1) == 1)))
    kept = kept + round_up.to(torch.int64)
    # biased exponent - 1 in the exponent field plus a significand that still holds its leading bit: the leading bit
    # adds the 1 back, a subnormal's (q = 1 - bias - dm) field is 0, a rounding carry moves into the exponent
    inf = ((1 << de) - 1) << dm
    mag = torch.clamp(q + dbias + dm - 1, min=0) << dm
    mag = torch.where(m == 0, torch.zeros_like(m), mag + kept)
    mag = torch.where(special | (mag >= inf), torch.full_like(mag, inf), mag)
    out = (sign << (de + dm)) | mag
    return torch.where(special & (frac != 0), torch.full_like(out, NAN), out)


def is_nan_bits(bits: torch.Tensor, t: torch.dtype) -> torch.Tensor:
    """Whether the ``t`` patterns in the low bits of ``bits`` are NaNs (integer arithmetic only)."""
    ne, nm, _ = FORMATS[t]
    x = bits.to(torch.int64)
    return (((x >> nm) & ((1 << ne) - 1)) == (1 << ne) - 1) & ((x & ((1 << nm) - 1)) != 0)


def all_16_bit_patterns(device="cpu") -> torch.Tensor:
    return torch.arange(1 << 16, dtype=torch.int64, device=device)


def structured_f32() -> np.ndarray:
    """F32 patterns (uint32) where conversions go wrong: for every exponent and both signs, the mantissas at, just
    below and just above the tie of every possible count of dropped bits (1 .. 23, covering BF16 from every binade and
    F16 from its normal and subnormal ranges), with even and odd kept parts; every F16 subnormal and normal-boundary
    value j * 2^-24 (j <= 2048) with the midpoints between them and their F32 neighbours; the F16 overflow edge
    65504 / 65519 / 65520 and neighbours; zeros, infinities, the F32 extremes and NaNs with payloads."""
    m = []
    for k in range(1, 24):  # k dropped bits: the tie is bit k - 1, the kept part's last bit is bit k
        tie = 1 << (k - 1)
        for low in (tie - 1, tie, tie + 1, 0, 1, (1 << k) - 1):
            for kept in (0, 1 << k, 3 << k, ((1 << 23) - 1) & ~((1 << k) - 1), 0x55555555 & ~((1 << k) - 1)):
                m.append((kept | low) & ((1 << 23) - 1))
    m = np.unique(np.array(m, np.uint32))
    exps = np.arange(256, dtype=np.uint32)
    grid = ((exps[:, None] << np.uint32(23)) | m[None, :]).reshape(-1)
    j = np.arange(0, 2049, dtype=np.float64)
    f16_grid = np.concatenate([j, j[:-1] + 0.5]) * 2.0**-24  # exact in F32
    edges = np.array([65504.0, 65519.0, 65520.0, 65535.0, 65536.0, 2.0**-14, 2.0**-24, 2.0**-25, 3 * 2.0**-26],
                     np.float64)
    near = np.concatenate([f16_grid, edges]).astype(np.float32).view(np.uint32)
    near = np.concatenate([near, near + np.uint32(1), near - np.uint32(1)])
    fixed = np.array([0, 1, 0x007FFFFF, 0x00800000, 0x7F7FFFFF, 0x7F800000, 0x7F800001, 0x7FC00000, 0x7FFFFFFF,
                      0x7FBFFFFF, 0x7F80FFFF, 0x7F810000, 0x7FFF0000, 0x477FE000, 0x477FEFFF, 0x477FF000, 0x477FF001,
                      0x47800000, 0x33000000, 0x33000001, 0x337FFFFF], np.uint32)
    pos = np.unique(np.concatenate([grid, near, fixed]))
    return np.concatenate([pos, pos | np.uint32(0x80000000)])


def random_f32(n: int, seed: int, device="cpu") -> torch.Tensor:
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randint(0, 1 << 32, (n,), dtype=torch.int64, device=device, generator=g)


def _as(bits: torch.Tensor, t: torch.dtype) -> torch.Tensor:
    """The ``t`` elements with these bit patterns (CPU)."""
    w = torch.finfo(t).bits
    signed = torch.where(bits >= 1 << (w - 1), bits - (1 << w), bits)
    return signed.to(INT_VIEW[t]).view(t)


def _bits(x: torch.Tensor) -> torch.Tensor:
    w = torch.finfo(x.dtype).bits
    return x.view(INT_VIEW[x.dtype]).to(torch.int64) & ((1 << w) - 1)


def _check_against_torch(bits: torch.Tensor, src: torch.dtype, dst: torch.dtype):
    ref = reference_cast(bits, src, dst)
    nan = is_nan_bits(bits, src)
    assert torch.equal(ref == NAN, nan)
    want = _bits(_as(bits, src).to(dst))
    bad = torch.nonzero(~nan & (ref != want)).flatten()[:8]
    assert not bad.numel(), (src, dst, [hex(v) for v in bits[bad].tolist()], [hex(v) for v in ref[bad].tolist()],
                             [hex(v) for v in want[bad].tolist()])
    # torch and the reference agree that a non-NaN never becomes a NaN
    assert not is_nan_bits(want[~nan], dst).any()
    return ref


SIXTEEN = [(s, d) for s in (torch.float16, torch.bfloat16) for d in (torch.float32, torch.float16, torch.bfloat16)
           if s != d]


@pytest.mark.parametrize("src,dst", SIXTEEN, ids=lambda t: str(t).split(".")[-1])
def test_every_16_bit_pattern_equals_torch_cpu(src, dst):
    bits = all_16_bit_patterns()
    ref = _check_against_torch(bits, src, dst)
    if dst == torch.float32:  # widening is exact: every non-NaN widens to a distinct value and back
        back = reference_cast(ref[ref != NAN], dst, src)
        assert torch.equal(back, bits[ref != NAN])


@pytest.mark.parametrize("dst", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_structured_f32_set_equals_torch_cpu_and_numpy(dst):
    raw = structured_f32()
    bits = torch.from_numpy(raw.astype(np.int64))
    ref = _check_against_torch(bits, torch.float32, dst)
    if dst == torch.float16:
        nan = ref == NAN
        with np.errstate(over="ignore"):  # overflow to infinity is what is being checked
            want = torch.from_numpy(raw.view(np.float32).astype(np.float16).view(np.uint16).astype(np.int64))
        assert torch.equal(ref[~nan], want[~nan])


def test_reference_spot_values():
    """Values fixed by the formats themselves, written out so the reference's arithmetic cannot drift with torch."""
    f32, f16, bf16 = torch.float32, torch.float16, torch.bfloat16

    def one(b, s, d):
        return int(reference_cast(torch.tensor([b]), s, d)[0])

    assert one(0x477FE000, f32, f16) == 0x7BFF  # 65504, the largest F16
    assert one(0x477FEFFF, f32, f16) == 0x7BFF  # 65519.99...: below the tie
    assert one(0x477FF000, f32, f16) == 0x7C00  # 65520: the tie rounds to even, which is 2^16: infinity
    assert one(0xC77FF000, f32, f16) == 0xFC00
    assert one(0x33800000, f32, f16) == 0x0001  # 2^-24, the smallest F16 subnormal
    assert one(0x33000000, f32, f16) == 0x0000  # 2^-25: the tie between 0 and 2^-24 goes to 0
    assert one(0x33000001, f32, f16) == 0x0001  # just above it
    assert one(0xB3000000, f32, f16) == 0x8000  # signed zero
    assert one(0x387FC000, f32, f16) == 0x03FF  # 2^-14 - 2^-24, the largest F16 subnormal
    assert one(0x387FE000, f32, f16) == 0x0400  # 2^-14 - 2^-25: the tie rounds up into the smallest normal
    assert one(0x3F808000, f32, bf16) == 0x3F80  # 1 + 2^-8: tie, even
    assert one(0x3F818000, f32, bf16) == 0x3F82  # 1 + 3 * 2^-8: tie, odd rounds up
    assert one(0x7F7FFFFF, f32, bf16) == 0x7F80  # F32 max rounds to infinity in BF16
    assert one(0x00000001, f32, bf16) == 0x0000  # F32 min subnormal
    assert one(0x00008000, f32, bf16) == 0x0000  # tie at BF16's smallest subnormal: even
    assert one(0x00018000, f32, bf16) == 0x0002
    assert one(0x0001, f16, f32) == 0x33800000
    assert one(0x03FF, f16, f32) == 0x387FC000
    assert one(0x7C00, f16, bf16) == 0x7F80
    assert one(0x0001, f16, bf16) == 0x3380
    assert one(0x7BFF, f16, bf16) == 0x4780  # 65504 = 0xFFE0 needs 11 bits: it rounds to 65536 in BF16
    assert one(0x4780, bf16, f16) == 0x7C00  # 65536: infinity
    assert one(0x477F, bf16, f16) == 0x7BF8  # 65280
    assert one(0x3380, bf16, f16) == 0x0001
    assert one(0x3300, bf16, f16) == 0x0000
    assert one(0x3340, bf16, f16) == 0x0001  # 1.5 * 2^-25 rounds up to 2^-24
    assert one(0x7FC0, bf16, f32) == NAN and one(0x7F800001, f32, f16) == NAN and one(0xFE00, f16, bf16) == NAN


def test_2_to_the_26_random_f32_patterns_equal_torch_cpu_and_numpy():
    for chunk in range(4):
        bits = random_f32(1 << 24, seed=100 + chunk)
        for dst in (torch.bfloat16, torch.float16):
            ref = _check_against_torch(bits, torch.float32, dst)
            if dst == torch.float16:
                nan = ref == NAN
                with np.errstate(over="ignore"):
                    want = _as(bits, torch.float32).numpy().astype(np.float16).view(np.uint16).astype(np.int64)
                assert torch.equal(ref[~nan], torch.from_numpy(want)[~nan])
