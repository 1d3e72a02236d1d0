"""The C ABI from a plain C99 host: tests/c/blob_host_check.c is compiled with gcc (-std=c99 -pedantic -Werror, so
both headers are valid C, not just C++), linked against libb200hash.so and driven with fake transport callbacks.
It mirrors how a cgo binding of go/blob.go's blobUpload would call the library."""
import base64
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest

from modal_client_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    _lib.build_library()
    out = str(tmp_path_factory.mktemp("c_host") / "blob_host_check")
    libdir = os.path.dirname(_lib.LIB_PATH)
    cmd = ["gcc", "-std=c99", "-O1", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c", "blob_host_check.c"), "-o", out, "-L", libdir, "-l:libb200hash.so",
           f"-Wl,-rpath,{libdir}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def _payload(seed: int, n: int) -> bytes:
    i = np.arange(n, dtype=np.uint64)
    return ((((i + np.uint64(seed)) & np.uint64(0xffffffff)) * np.uint64(2654435761) & np.uint64(0xffffffff))
            >> np.uint64(24)).astype(np.uint8).tobytes()


def test_blob_header_declares_what_the_library_exports():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b200blob.h")).read(), flags=re.S)
    declared = sorted(set(re.findall(r"\b(b200blob_[a-z0-9_]+)\s*\(", text)))
    assert declared == ["b200blob_hashes_many", "b200blob_should_upload", "b200blob_upload", "b200blob_upload_many"]
    lib = _lib.load_library()
    for sym in declared:
        assert hasattr(lib, sym), sym


def test_c_host_compiles_and_fails_loudly_without_gpu(exe):
    r = subprocess.run([exe, "nogpu"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "OK nogpu" in r.stdout, r.stdout + r.stderr
    assert "sm_90a" in r.stdout


@pytest.mark.gpu
def test_c_host_blob_upload_matches_hashlib(exe):
    r = subprocess.run([exe, "run"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "OK run" in r.stdout, r.stdout + r.stderr
    lines = r.stdout.splitlines()
    seen = 0
    for ln in lines:
        if ln.startswith("hashes "):
            _, seed, n, md5_b64, sha_b64, _id = ln.split()
            data = _payload(int(seed), int(n))
            assert md5_b64 == base64.b64encode(hashlib.md5(data).digest()).decode()      # go/blob.go:51,53
            assert sha_b64 == base64.b64encode(hashlib.sha256(data).digest()).decode()   # go/blob.go:52,54
            seen += 1
    assert seen == 8 + 9
    text = r.stdout
    assert "multipart_error Function input size exceeds multipart upload threshold, unsupported by this SDK version" in text
    assert "no_url_error missing upload URL in BlobCreate response" in text
    assert "create_error failed to create blob: rpc unavailable" in text
    assert "put_error failed blob upload: 500" in text
    launches = int(re.search(r"many_launches (\d+)", text).group(1))
    assert launches <= 6  # 300 payloads: ONE batch (3 plan kernels + chain + lane_hash launches), not 300 hash calls


# ---------------------------------------------------------------------------- JS SDK: the N-API addon (js/src/blob.ts)


@pytest.fixture(scope="module")
def napi_exe(tmp_path_factory):
    """bindings/node/b200hash_napi.c compiled as strict C99 against tests/c/node_api.h (stand-in for the Node-API subset
    it uses; Node itself is not in this image) together with the C driver that plays Node's part."""
    _lib.build_library()
    out = str(tmp_path_factory.mktemp("napi") / "napi_host_check")
    libdir = os.path.dirname(_lib.LIB_PATH)
    inc = ["-I", os.path.join(ROOT, "tests", "c"), "-I", os.path.join(ROOT, "include")]
    addon = os.path.join(ROOT, "bindings", "node", "b200hash_napi.c")
    strict = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-fsyntax-only", *inc, addon],
                            capture_output=True, text=True)
    assert strict.returncode == 0, strict.stderr
    cmd = ["gcc", "-std=c99", "-D_POSIX_C_SOURCE=200809L", "-O1", "-Wall", "-Wextra", "-Werror", *inc,
           os.path.join(ROOT, "tests", "c", "napi_host_check.c"), addon, "-o", out, "-L", libdir, "-l:libb200hash.so",
           f"-Wl,-rpath,{libdir}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def _js_payload(i: int, n: int) -> bytes:
    k = np.arange(n, dtype=np.uint64)
    return ((np.uint64(i * 131) + k * np.uint64(7) + np.uint64(1)) & np.uint64(0xff)).astype(np.uint8).tobytes()


def test_napi_addon_compiles_and_throws_without_gpu(napi_exe):
    import json

    r = subprocess.run([napi_exe, "10", "20"], capture_output=True, text=True, timeout=120)
    out = json.loads(r.stdout)
    if "error" in out:  # no GPU here: the JS side sees an exception, never a CPU digest
        assert "no CPU fallback" in out["error"] and r.returncode == 1
    else:
        assert len(out["md5"]) == 2


@pytest.mark.gpu
def test_napi_addon_hashes_many_matches_node_crypto_semantics(napi_exe):
    """exports.hashesMany(Uint8Array[]) == createHash(..).update(data).digest("base64") per payload
    (js/src/blob.ts:35-36), in one GPU batch; exports.shouldUpload is the strict 2 MiB gate."""
    import json

    sizes = [0, 1, 55, 64, 1000, 65536, 300001, 2 * 1024 * 1024 + 1]
    r = subprocess.run([napi_exe, *map(str, sizes)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    out = json.loads(r.stdout)
    for i, n in enumerate(sizes):
        data = _js_payload(i, n)
        assert out["md5"][i] == base64.b64encode(hashlib.md5(data).digest()).decode()
        assert out["sha256"][i] == base64.b64encode(hashlib.sha256(data).digest()).decode()
    assert out["should_upload_2MiB"] is False and out["should_upload_2MiB_plus_1"] is True
    assert out["throws_on_non_array"] is True


@pytest.mark.parametrize("sanitize", [False, True], ids=["plain", "tsan"])
def test_packer_team_hands_every_grain_out_exactly_once(tmp_path, sanitize):
    """modal_client_b200/csrc/b200pack_team.h (the parked packer / reader threads of a context) driven by
    tests/c/pack_team_check.cpp: thousands of jobs of the grain-counter kind, changing team sizes, clean shutdown --
    once as a plain build, once under ThreadSanitizer (skipped where the toolchain has no libtsan)."""
    out = str(tmp_path / "pack_team_check")
    cmd = ["g++", "-std=c++17", "-pthread", "-Wall", "-Wextra", "-Werror"]
    cmd += ["-O1", "-g", "-fsanitize=thread"] if sanitize else ["-O2"]
    cmd += [os.path.join(ROOT, "tests", "c", "pack_team_check.cpp"), "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if sanitize and r.returncode != 0 and ("tsan" in r.stderr.lower() or "sanitize" in r.stderr.lower()):
        pytest.skip("ThreadSanitizer runtime not available: " + r.stderr.strip().splitlines()[-1])
    assert r.returncode == 0, r.stderr
    r = subprocess.run([out, "2000" if sanitize else "20000"], capture_output=True, text=True, timeout=600)
    if sanitize and "FATAL: ThreadSanitizer" in r.stderr:  # e.g. an address-space layout the runtime refuses
        pytest.skip(r.stderr.strip().splitlines()[0])
    assert r.returncode == 0 and "PACK TEAM OK" in r.stdout, r.stdout + r.stderr
    assert "WARNING: ThreadSanitizer" not in r.stderr, r.stderr[-3000:]
