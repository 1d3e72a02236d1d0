"""Drop-in for the reference's ``modal/_utils/hash_utils.py`` with the arithmetic on the GPU.

Same names, signatures, return types and stream semantics as the reference
(py/modal/_utils/hash_utils.py:14-101); the hashlib objects are replaced by libb200hash calls:

* ``bytes`` input  -> one message through ``b200h_hash_batch_host`` (both digests in one read);
* stream input     -> ``b200h_stream_*``: read from the current position to EOF in ``HASH_CHUNK_SIZE``
  pieces, restore the position afterwards (reference :20,:29), reject non-bytes chunks (:23-24).

``get_upload_hashes_many`` is the batched entry point the accelerated callers use (map input pump,
Volume.batch_upload): N payloads, one GPU batch, N ``UploadHashes``.
"""
from __future__ import annotations

import base64
import binascii
import dataclasses
import time
from collections.abc import Callable, Sequence
from typing import BinaryIO

from ._backend import get_context
from ._lib import MD5, SHA256
from ._logging import logger

HASH_CHUNK_SIZE = 65536  # module global on purpose: the reference's tests patch it by name


def _update(hashers: Sequence[Callable[[bytes], None]], data: bytes | BinaryIO) -> None:
    """Feed ``data`` to every updater in ``hashers`` (reference :14-29)."""
    if isinstance(data, bytes):
        for push in hashers:
            push(data)
        return
    assert not isinstance(data, (bytearray, memoryview))
    start = data.tell()
    while True:
        chunk = data.read(HASH_CHUNK_SIZE)
        if not isinstance(chunk, bytes):
            raise ValueError(f"Only accepts bytes or byte buffer objects, not {type(chunk)} buffers")
        if len(chunk) == 0:
            break
        for push in hashers:
            push(chunk)
    data.seek(start)


def _digests(data: bytes | BinaryIO, flags: int) -> tuple[bytes | None, bytes | None]:
    """(sha256 raw | None, md5 raw | None) of one message, computed on the GPU."""
    ctx = get_context()
    if isinstance(data, bytes):
        sha, md5, _ = ctx.hash_buffers([data], flags)
        return (sha[0].tobytes() if sha is not None else None, md5[0].tobytes() if md5 is not None else None)
    stream = ctx.stream(flags)
    try:
        _update([stream.update], data)
        return stream.digests()
    finally:
        stream.close()


def get_sha256_hex(data: bytes | BinaryIO) -> str:
    t0 = time.monotonic()
    sha, _ = _digests(data, SHA256)
    logger.debug("get_sha256_hex took %.3fs", time.monotonic() - t0)
    return sha.hex()


def get_sha256_base64(data: bytes | BinaryIO) -> str:
    t0 = time.monotonic()
    sha, _ = _digests(data, SHA256)
    logger.debug("get_sha256_base64 took %.3fs", time.monotonic() - t0)
    return base64.b64encode(sha).decode("ascii")


def get_md5_base64(data: bytes | BinaryIO) -> str:
    t0 = time.monotonic()
    _, md5 = _digests(data, MD5)
    logger.debug("get_md5_base64 took %.3fs", time.monotonic() - t0)
    return base64.b64encode(md5).decode("utf-8")


@dataclasses.dataclass
class UploadHashes:
    md5_base64: str
    sha256_base64: str

    def md5_hex(self) -> str:
        return base64.b64decode(self.md5_base64).hex()

    def sha256_hex(self) -> str:
        return base64.b64decode(self.sha256_base64).hex()


def _b64(raw: bytes) -> str:
    return binascii.b2a_base64(raw, newline=False).decode("ascii")


class _UploadHashesRaw(UploadHashes):
    """UploadHashes that still knows the raw digests it was formatted from (rows of a GPU digest table), so the
    upload code does not have to decode the base64 again to compare ETags."""

    md5_raw: bytes | None = None
    sha256_raw: bytes | None = None

    def __init__(self, md5_base64: str, sha256_base64: str, md5_raw: bytes | None = None, sha256_raw: bytes | None = None):
        self.md5_base64 = md5_base64
        self.sha256_base64 = sha256_base64
        self.md5_raw = md5_raw
        self.sha256_raw = sha256_raw

    def md5_hex(self) -> str:
        return self.md5_raw.hex() if self.md5_raw is not None else super().md5_hex()

    def sha256_hex(self) -> str:
        return self.sha256_raw.hex() if self.sha256_raw is not None else super().sha256_hex()


def get_upload_hashes(
    data: bytes | BinaryIO, sha256_hex: str | None = None, md5_hex: str | None = None
) -> UploadHashes:
    """Both upload digests in a single pass over ``data``; a digest supplied by the caller is passed
    through (hex -> base64) and NOT recomputed (reference :74-93)."""
    t0 = time.monotonic()
    flags = (0 if sha256_hex else SHA256) | (0 if md5_hex else MD5)
    sha_raw = md5_raw = None
    if flags:
        sha_raw, md5_raw = _digests(data, flags)
    out = UploadHashes(
        md5_base64=_b64(bytes.fromhex(md5_hex) if md5_hex else md5_raw),
        sha256_base64=_b64(bytes.fromhex(sha256_hex) if sha256_hex else sha_raw),
    )
    logger.debug("get_upload_hashes took %.3fs (flags=%d)", time.monotonic() - t0, flags)
    return out


def _b64_rows(table, width: int) -> str | None:
    """base64 of every ``width``-byte row of a uint8[n, width] table in ONE C call, rows back to back and each
    complete with its ``=`` padding: rows are zero-padded to a multiple of 3 bytes, so row i occupies a fixed slice
    of the result whose leading characters are exactly the row's own base64 (the padding bits are zero either way);
    the characters that stand for the pad bytes are then overwritten with ``=`` for all rows at once."""
    if table is None:
        return None
    import numpy as np

    n = table.shape[0]
    padded = -(-width // 3) * 3
    buf = np.zeros((n, padded), np.uint8)
    buf[:, :width] = table
    text = np.frombuffer(binascii.b2a_base64(buf, newline=False), np.uint8).reshape(n, padded // 3 * 4).copy()
    if padded != width:
        text[:, -(padded - width):] = 0x3D  # '='
    return text.tobytes().decode("ascii")


class _UploadHashesView(Sequence):
    """Read-only sequence of ``UploadHashes`` over a digest table; rows are formatted on access (base64 of the whole
    table is one C call, a row is two string slices), so a batch of 10^5..10^6 payloads pays well under 1 us per row."""

    def __init__(self, sha, md5, n: int):
        self._sha, self._md5, self._n = sha, md5, n
        self._sha64 = _b64_rows(sha, 32)  # 44 chars per row
        self._md564 = _b64_rows(md5, 16)  # 24 chars per row
        self._sha_bytes = sha.tobytes() if sha is not None else None
        self._md5_bytes = md5.tobytes() if md5 is not None else None

    def __len__(self) -> int:
        return self._n

    def columns(self) -> tuple[str | None, str, bytes | None]:
        """(md5 base64 text, 24 chars per row | None, sha256 base64 text, 44 chars per row, raw md5 bytes, 16 per row |
        None): for callers that walk every row and do not want an object per row."""
        return self._md564, self._sha64, self._md5_bytes

    def __getitem__(self, i):
        if i.__class__ is not int:
            if isinstance(i, slice):
                return [self[j] for j in range(*i.indices(self._n))]
            i = int(i)
        if i < 0:
            i += self._n
        if not 0 <= i < self._n:
            raise IndexError(i)
        if self._md564 is None:
            return _UploadHashesRaw("", self._sha64[44 * i : 44 * i + 44], None, self._sha_bytes[32 * i : 32 * i + 32])
        return _UploadHashesRaw(self._md564[24 * i : 24 * i + 24], self._sha64[44 * i : 44 * i + 44],
                                self._md5_bytes[16 * i : 16 * i + 16], self._sha_bytes[32 * i : 32 * i + 32])


def get_upload_hashes_many(payloads: Sequence[bytes], *, want_md5: bool = True, ctx=None) -> Sequence[UploadHashes]:
    """N in-memory payloads -> N UploadHashes in ONE GPU batch.  This replaces the serial
    ``get_upload_hashes(payload)`` loop the map pump runs on its event-loop thread
    (py/modal/_utils/blob_utils.py:345 under parallel_map.py:139) and Go's per-call md5.Sum/sha256.Sum256
    (go/blob.go:51-52).  ``want_md5=False`` leaves md5_base64 empty (callers that hold a placeholder)."""
    if not payloads:
        return []
    flags = SHA256 | (MD5 if want_md5 else 0)
    sha, md5, _ = (ctx or get_context()).hash_buffers(payloads, flags)
    return _UploadHashesView(sha, md5, len(payloads))
