"""CPU: the C-ABI library loads, exports every symbol include/b200hash.h declares, and refuses to
work (loudly, no CPU fallback) when no GPU is visible."""
import os
import re

import pytest

from modal_client_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "b200hash.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200h_[a-z0-9_]+)\s*\(", text)))


def test_header_and_binding_agree():
    assert _declared_symbols() == sorted(_lib.ABI_SYMBOLS)


def test_library_exports_every_declared_symbol():
    _lib.build_library()
    lib = _lib.load_library()
    for sym in _declared_symbols():
        assert hasattr(lib, sym), sym
    assert b"sm_90a" in lib.b200h_version()


def test_no_cpu_fallback_without_gpu():
    lib = _lib.load_library()
    if lib.b200h_device_count() > 0:
        pytest.skip("a GPU is visible")
    with pytest.raises(_lib.B200HashError) as ei:
        _lib.Context(0)
    assert "no CPU fallback" in str(ei.value) or "CUDA" in str(ei.value)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "modal_client_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert not re.search(r"^\s*(from|import)\s+hashlib\b", src, flags=re.M), f


@pytest.mark.parametrize("isa", ["avx512", "avx2", "plain"])
def test_stream_copy_is_a_memcpy_for_every_size_and_alignment(isa):
    """b200h_stream_copy (csrc/b200pack_copy.cpp) fills the pinned staging ring of every *_host entry point: a wrong
    byte here is a wrong digest on the GPU.  Each variant -- capped with B200H_COPY_ISA; the dispatch is decided once
    per process, hence the subprocess -- must copy exactly n bytes for every size class (below / above the 4 KiB
    streaming threshold, non-multiples of the unroll) and every source / destination misalignment, and must not touch
    the bytes around the destination."""
    import subprocess
    import sys

    code = r"""
import ctypes, sys
import numpy as np
sys.path.insert(0, %r)
from modal_client_b200 import _lib
L = _lib.load_library()
got = L.b200h_stream_copy_isa().decode()
rng = np.random.default_rng(7)
src = rng.integers(0, 256, 3 << 20, dtype=np.uint8)
dst = np.empty(3 << 20, np.uint8)
sizes = [0, 1, 31, 63, 64, 4095, 4096, 4097, 4096 + 127, 4096 + 128, 4096 + 255, 4096 + 256, 4096 + 257, 65536 + 3,
         262144, 262144 + 17, 1 << 20, (1 << 20) + 255, (2 << 20) + 511]
for n in sizes:
    for so in (0, 1, 13, 32, 63):
        for do in (64, 65, 77, 96, 127):
            dst[:] = 0xA5
            L.b200h_stream_copy(ctypes.c_void_p(dst.ctypes.data + do), ctypes.c_void_p(src.ctypes.data + so), n)
            assert np.array_equal(dst[do:do + n], src[so:so + n]), (n, so, do)
            assert (dst[:do] == 0xA5).all() and (dst[do + n:do + n + 512] == 0xA5).all(), (n, so, do)
print(got)
""" % (os.path.dirname(os.path.dirname(os.path.abspath(__file__))),)
    env = dict(os.environ, B200H_COPY_ISA=isa)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    got = out.stdout.strip().splitlines()[-1]
    assert got in ("avx512", "avx2", "plain")
    order = ["plain", "avx2", "avx512"]
    assert order.index(got) <= order.index(isa)  # the cap is honoured; a CPU without the ISA falls further back



def test_hash_buffers_passes_the_payloads_own_addresses(monkeypatch):
    """hash_buffers hands the library absolute addresses of the bytes objects' payloads (no copy, no numpy view per
    payload): what it passes must read back as the payloads themselves."""
    import ctypes

    import numpy as np

    seen = {}

    def capture(self, base, offsets, lengths, flags=3):
        seen["base"], seen["off"], seen["len"] = base, np.array(offsets), np.array(lengths)
        return None, None, None

    monkeypatch.setattr(_lib.Context, "hash_batch_host", capture)
    ctx = object.__new__(_lib.Context)  # no GPU needed: only the argument marshalling is under test
    bufs = [bytes([i % 251]) * (i * 37 % 500) + b"x" for i in range(300)]
    ctx.hash_buffers(bufs)
    assert seen["base"] is None and seen["off"].dtype == np.uint64 and seen["len"].dtype == np.uint64
    assert [ctypes.string_at(int(o), int(n)) for o, n in zip(seen["off"], seen["len"])] == bufs
    mixed = [b"abc", bytearray(b"defg"), memoryview(b"hi")]
    ctx.hash_buffers(mixed)  # anything that is not plain bytes goes through numpy views
    assert [ctypes.string_at(int(o), int(n)) for o, n in zip(seen["off"], seen["len"])] == [bytes(m) for m in mixed]


@pytest.mark.parametrize("threads,slot_mib", [(1, 32), (2, 8), (3, 13), (8, 32), (16, 64)])
def test_packer_team_gathers_every_message_to_its_place(threads, slot_mib):
    """b200h_pack_preview runs the packer team of the *_host entry points (pack_parallel: grains handed out from a shared
    counter) without a GPU.  Whatever the team size and slot size, every message must land byte for byte at its packed
    offset (next multiple of 16), across grain and slot boundaries, for empty, tiny and multi-MiB messages, unaligned
    sources, and both addressing forms (base + offset, absolute addresses)."""
    import numpy as np

    rng = np.random.default_rng(threads * 100 + slot_mib)
    lens = np.concatenate([
        rng.integers(0, 64, 200), rng.integers(64, 70_000, 400), rng.integers(200_000, 3_000_000, 40),
        [0, 1, 15, 16, 17, (1 << 20) - 1, 1 << 20, (1 << 20) + 1, 5 << 20],
    ]).astype(np.uint64)
    rng.shuffle(lens)
    gaps = rng.integers(0, 40, lens.size).astype(np.uint64)
    offs = (np.concatenate([[0], np.cumsum(lens + gaps)])[:-1] + np.uint64(3)).astype(np.uint64)
    src = rng.integers(0, 256, int(offs[-1] + lens[-1]) + 64, dtype=np.uint8)
    packed, doff = _lib.pack_preview(src, offs, lens, threads=threads, slot_bytes=slot_mib << 20)
    expect_off = np.concatenate([[0], np.cumsum((lens + np.uint64(15)) & ~np.uint64(15))])[:-1].astype(np.uint64)
    assert np.array_equal(doff, expect_off)
    for i in range(lens.size):
        a, n, s = int(doff[i]), int(lens[i]), int(offs[i])
        assert np.array_equal(packed[a:a + n], src[s:s + n]), i
    # absolute addresses (what hash_buffers passes for Python bytes objects)
    packed2, doff2 = _lib.pack_preview(None, offs + np.uint64(src.ctypes.data), lens, threads=threads, slot_bytes=slot_mib << 20)
    assert np.array_equal(doff2, doff)
    for i in range(0, lens.size, 7):
        a, n = int(doff[i]), int(lens[i])
        assert np.array_equal(packed2[a:a + n], packed[a:a + n])
    with pytest.raises(_lib.B200HashError):
        _lib.pack_preview(src, offs, lens, threads=threads, dst=np.empty(1024, np.uint8))  # destination too small


def test_packer_team_survives_many_slots_and_concurrent_callers():
    """The packer threads are started once and parked between slots (PackTeam): hundreds of wake-ups, a team that grows
    between calls, and several callers at once (each with its own team, like contexts) must neither lose a byte nor hang."""
    import threading

    import numpy as np

    rng = np.random.default_rng(3)
    lens = rng.integers(100_000, 400_000, 600).astype(np.uint64)  # ~150 MB
    offs = np.concatenate([[0], np.cumsum(lens + np.uint64(5))])[:-1].astype(np.uint64)
    src = rng.integers(0, 256, int(offs[-1] + lens[-1]) + 16, dtype=np.uint8)
    expect_off = np.concatenate([[0], np.cumsum((lens + np.uint64(15)) & ~np.uint64(15))])[:-1]
    errors = []

    def caller(seed):
        try:
            for rep in range(6):
                threads = [2, 5, 8, 3, 16, 4][(rep + seed) % 6]
                packed, doff = _lib.pack_preview(src, offs, lens, threads=threads, slot_bytes=(8 + 8 * ((rep + seed) % 3)) << 20)
                assert np.array_equal(doff, expect_off)
                for i in range(seed % 7, lens.size, 7):
                    a, n, s = int(doff[i]), int(lens[i]), int(offs[i])
                    assert np.array_equal(packed[a:a + n], src[s:s + n]), (seed, rep, i)
        except BaseException as exc:  # noqa: BLE001 - reported by the main thread
            errors.append(exc)

    ths = [threading.Thread(target=caller, args=(k,)) for k in range(4)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=240)
    assert not any(t.is_alive() for t in ths), "a packer team hung"
    assert not errors, errors[0]
