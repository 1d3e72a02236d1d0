"""Drop-in for the hashing / chunking half of the reference's ``modal/_utils/blob_utils.py``.

Same public names, size classes, thresholds and integrity checks as the reference
(py/modal/_utils/blob_utils.py), with every digest produced by libb200hash on the GPU:

=============================  ===========================================================================
reference (file:line)          here
=============================  ===========================================================================
``_get_file_upload_spec``      same semantics per file; ``get_file_upload_specs`` hashes a whole *list* of
  :446-487                     files in one GPU batch (what ``Volume.batch_upload`` v1 / ``Mount`` need)
``_gather_blocks`` … :622-705  one ``b200h_hash_fixed_parts(TRIM_ZEROS)`` call per file: the zero-trim scan and
                               the SHA-256 of every 8 MiB block run on the device, the file is read ONCE
``perform_multipart_upload``   all part MD5s + the md5-of-md5s ETag come from one GPU call before any byte is
  :159-234                     sent; the per-chunk CPU re-hash inside the payload disappears
``_blob_upload`` … :271-374    unchanged control flow (BlobCreate -> single PUT | multipart), GPU digests
=============================  ===========================================================================

Module constants stay patchable module globals read at call time, because the reference's tests patch
them by dotted name (py/test/blob_test.py:57, py/test/volume_test.py:489).
"""
from __future__ import annotations

import asyncio
import dataclasses
import functools
import gc
import mmap
import os
import platform
import time
from collections.abc import Callable, Sequence
from contextlib import AbstractContextManager, asynccontextmanager, contextmanager
from io import BytesIO, FileIO
from pathlib import Path, PurePosixPath
from typing import Any, BinaryIO, ContextManager
from urllib.parse import urlparse

import numpy as np

from . import _lib, _wire, hash_utils
from ._backend import get_context
from ._logging import logger
from ._wire import BlobCreateRequest
from .async_utils import asyncnullcontext, bounded_map, gather_cancel_on_error, retry
from .bytes_io_segment_payload import BytesIOSegmentPayload, KnownBytesBody
from .device_file import DeviceFile, hash_parts_many
from .exception import ExecutionError
from .hash_utils import UploadHashes, get_upload_hashes
from .http_utils import ClientSessionRegistry

MAX_OBJECT_SIZE_BYTES = 2 * 1024 * 1024  # function inputs/outputs above this go to blob storage
MAX_ASYNC_OBJECT_SIZE_BYTES = 8 * 1024  # ... for async (spawn) calls
LARGE_FILE_LIMIT = 4 * 1024 * 1024  # files at least this big are uploaded as blobs
BLOB_MAX_PARALLELISM = 20
DEFAULT_SEGMENT_CHUNK_SIZE = 2**24
MULTIPART_UPLOAD_THRESHOLD = 1024**3  # above this no whole-file MD5 is computed (placeholder instead)
MULTIPART_INFLIGHT_BYTES_MAX = 2 * 1024**3
MULTIPART_INFLIGHT_BYTES_MIN = 256 * 1024 * 1024
MULTIPART_INFLIGHT_MEMORY_FRACTION = 0.5
BLOCK_SIZE: int = 8 * 1024 * 1024  # volumefs2 block
SMALL_FILE_INLINE_LIMIT = 256 * 1024  # below this the content is cached in the spec
_MD5_PLACEHOLDER = "baadbaad" * 4


# --------------------------------------------------------------------------------------- byte budget


class _ByteBudget:
    """Caps the bytes in flight across concurrent part uploads (reference :66-91)."""

    def __init__(self, total: int):
        self._total = total
        self._available = total
        self._cond = asyncio.Condition()

    @classmethod
    def from_system_memory(cls) -> "_ByteBudget":
        return cls(_get_multipart_inflight_budget())

    @asynccontextmanager
    async def acquire(self, n: int):
        async with self._cond:
            # a request larger than the whole budget is admitted once nothing else is in flight
            await self._cond.wait_for(lambda: self._available >= min(n, self._total))
            self._available -= n
        try:
            yield
        finally:
            async with self._cond:
                self._available += n
                self._cond.notify_all()


def _get_multipart_inflight_budget() -> int:
    try:
        import psutil

        available = psutil.virtual_memory().available
    except Exception:
        try:
            available = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
        except (AttributeError, ValueError, OSError):
            return MULTIPART_INFLIGHT_BYTES_MIN
    want = int(available * MULTIPART_INFLIGHT_MEMORY_FRACTION)
    return min(max(want, MULTIPART_INFLIGHT_BYTES_MIN), MULTIPART_INFLIGHT_BYTES_MAX)


# ------------------------------------------------------------------------------ views of file contents


@contextmanager
def _readonly_view(fp: BinaryIO):
    """uint8 ndarray over the whole content of ``fp`` without copying when possible:
    BytesIO -> its buffer; real file -> a private read-only mmap; anything else -> one read()."""
    if isinstance(fp, BytesIO):
        buf = fp.getbuffer()
        arr = np.frombuffer(buf, dtype=np.uint8)
        try:
            yield arr
        finally:
            del arr
            buf.release()  # callers drop their references first (see _with_view)
        return
    try:
        fd = fp.fileno()
        size = os.fstat(fd).st_size
    except (OSError, AttributeError, ValueError):
        fd, size = None, 0
    if fd is not None and size > 0:
        mm = mmap.mmap(fd, 0, access=mmap.ACCESS_READ)
        try:
            arr = np.frombuffer(mm, dtype=np.uint8)
            yield arr
            del arr
        finally:
            mm.close()
        return
    pos = fp.tell()
    fp.seek(0)
    data = fp.read()
    fp.seek(pos)
    yield np.frombuffer(data, dtype=np.uint8)


def _with_view(fp: BinaryIO, fn):
    """fn(view) over the content of ``fp``; the view is dropped before the underlying buffer is released,
    so BytesIO objects stay closable/resizable afterwards."""
    with _readonly_view(fp) as view:
        try:
            return fn(view)
        finally:
            del view


# ------------------------------------------------------------------------------------ single-part PUT


@retry(n_attempts=3, base_delay=0.3, attempt_timeout=None)
async def _upload_to_s3_url(
    upload_url,
    payload,
    content_md5_b64: str | None = None,
    content_type: str | None = "application/octet-stream",
) -> str:
    """PUT one payload; returns the object's ETag after checking it against the local MD5
    (reference :110-156: S3's single-part ETag is the quoted MD5 hex of the body)."""
    with payload.reset_on_error():
        body = payload.as_payload() if isinstance(payload, KnownBytesBody) else payload
        headers = {}
        if content_md5_b64 and use_md5(upload_url):
            headers["Content-MD5"] = content_md5_b64
        if content_type:
            headers["Content-Type"] = content_type
        async with ClientSessionRegistry.get_session().put(
            upload_url, data=body, headers=headers, skip_auto_headers=["content-type"] if content_type is None else []
        ) as resp:
            if resp.status == 503:  # S3 SlowDown
                logger.debug("Received SlowDown signal from S3, sleeping for 1 second before retrying.")
                await asyncio.sleep(1)
            if resp.status != 200:
                try:
                    text = await resp.text()
                except Exception:
                    text = "<no body>"
                raise ExecutionError(f"Put to url {upload_url} failed with status {resp.status}: {text}")
            etag = resp.headers["ETag"].strip()
            if etag[:2] in ("W/", "w/"):
                etag = etag[2:]
            if len(etag) >= 2 and etag[0] == '"' and etag[-1] == '"':
                etag = etag[1:-1]
            local_md5_hex = payload.md5_checksum().hexdigest()
            if local_md5_hex != etag:
                raise ExecutionError(f"Local data and remote data checksum mismatch ({local_md5_hex} vs {etag})")
            return etag


# ------------------------------------------------------------------------------------------ multipart


def multipart_part_digests(data, part_length: int) -> tuple[list[bytes], str]:
    """All part MD5s of ``data`` split every ``part_length`` bytes plus the expected combined ETag
    ``md5(md5_0 || md5_1 || ...).hex() + "-<n>"`` -- one GPU call (reference :194-219 does n hashlib passes
    on executor threads and one more on the loop thread)."""
    _, md5, _, etag = get_context().hash_fixed_parts(data, part_length, _lib.MD5, want_etag=True)
    parts = [md5[i].tobytes() for i in range(len(md5))]
    return parts, f"{etag.hex()}-{len(parts)}"


async def perform_multipart_upload(
    data_file: BinaryIO | BytesIO | FileIO,
    *,
    content_length: int,
    max_part_size: int,
    part_urls: list[str],
    completion_url: str,
    upload_chunk_size: int = DEFAULT_SEGMENT_CHUNK_SIZE,
    progress_report_cb: Callable | None = None,
    byte_budget: _ByteBudget | None = None,
) -> None:
    # 1. hash every part on the GPU before sending anything
    start_pos = data_file.tell() if isinstance(data_file, BytesIO) else 0
    part_md5, expected_etag = await asyncio.to_thread(
        _with_view, data_file,
        lambda whole: multipart_part_digests(whole[start_pos : start_pos + content_length], max_part_size))
    if len(part_md5) > len(part_urls):
        raise ExecutionError(f"{len(part_md5)} parts but only {len(part_urls)} part URLs")

    # 2. one independent reader per part (no shared file position)
    if isinstance(data_file, BytesIO):
        view = data_file.getbuffer()
        readers: list[BinaryIO] = [BytesIO(view) for _ in part_urls]
        for rdr in readers:
            rdr.seek(start_pos)
    elif isinstance(data_file, DeviceFile):  # no file name to open again: readers over the same device bytes
        readers = [data_file.reopen() for _ in part_urls]
    else:
        readers = [open(data_file.name, "rb") for _ in part_urls]

    async def send(url: str, payload) -> str:
        async with byte_budget.acquire(4 * payload.chunk_size) if byte_budget else asyncnullcontext():
            return await _upload_to_s3_url(url, payload=payload, content_type=None)

    jobs, offset, left = [], 0, content_length
    for i, (rdr, url) in enumerate(zip(readers, part_urls)):
        n = min(left, max_part_size)
        payload = BytesIOSegmentPayload(rdr, segment_start=offset, segment_length=n, chunk_size=upload_chunk_size,
                                        progress_report_cb=progress_report_cb,
                                        md5_digest=part_md5[i] if i < len(part_md5) else None)
        jobs.append(send(url, payload))
        offset += n
        left -= n
    try:
        part_etags = await gather_cancel_on_error(*jobs)
    finally:
        if not isinstance(data_file, BytesIO):
            for rdr in readers:
                rdr.close()

    xml = ["<CompleteMultipartUpload>"]
    for number, etag in enumerate(part_etags, 1):
        xml.append(f'<Part>\n<PartNumber>{number}</PartNumber>\n<ETag>"{etag}"</ETag>\n</Part>')
    xml.append("</CompleteMultipartUpload>")
    # each part's ETag was already checked against the GPU digest in _upload_to_s3_url, so the device-side
    # md5-of-md5s is exactly what the store must report for the assembled object
    if len(part_md5) != len(part_etags):
        expected_etag = _etag_from_part_hexes(part_etags)
    resp = await ClientSessionRegistry.get_session().post(
        completion_url, data="\n".join(xml).encode("ascii"), skip_auto_headers=["content-type"]
    )
    if resp.status != 200:
        try:
            msg = await resp.text()
        except Exception:
            msg = "<no body>"
        raise ExecutionError(f"Error when completing multipart upload: {resp.status}\n{msg}")
    body_text = await resp.text()
    if expected_etag not in body_text:
        raise ExecutionError(f"Hash mismatch on multipart upload assembly: {expected_etag} not in {body_text}")


def _etag_from_part_hexes(part_etags: Sequence[str]) -> str:
    raw = b"".join(bytes.fromhex(e) for e in part_etags)
    _, md5, _ = get_context().hash_buffers([raw], _lib.MD5)
    return f"{md5[0].tobytes().hex()}-{len(part_etags)}"


# ---------------------------------------------------------------------------------------- blob upload


def get_content_length(data: BinaryIO) -> int:
    """Bytes from the current position to the end of the stream."""
    here = data.tell()
    end = data.seek(0, os.SEEK_END)
    data.seek(here)
    return end - here


async def _blob_upload_with_fallback(items, blob_ids: list[str], callback, content_length: int) -> tuple[str, bool, int]:
    """Try each storage provider in order; report whether R2 failed and the R2 throughput (reference :246-268)."""
    r2_failed, r2_bps = False, 0
    for idx, (item, blob_id) in enumerate(zip(items, blob_ids)):
        is_r2 = blob_id.endswith(":r2")
        try:
            t0 = time.monotonic_ns()
            await callback(item)
            if is_r2:
                r2_bps = (content_length * 1_000_000_000) // max(time.monotonic_ns() - t0, 1)
            return blob_id, r2_failed, r2_bps
        except Exception:
            r2_failed = r2_failed or is_r2
            if idx == len(items) - 1:
                raise
    raise ExecutionError("Failed to upload blob")


async def _blob_upload(
    upload_hashes: UploadHashes,
    data: bytes | BinaryIO,
    stub,
    progress_report_cb: Callable | None = None,
    byte_budget: _ByteBudget | None = None,
    _blob_create_response=None,
) -> tuple[str, bool, int]:
    """BlobCreate with the precomputed digests, then a single PUT or a multipart upload (reference :271-335).
    The map pump calls this once per blobified input, 10^5 times per map: a ``bytes`` payload is not wrapped in a
    reader (nor is its aiohttp payload object built) before a PUT actually needs one."""
    if isinstance(data, bytes):
        reader, content_length = None, len(data)
    else:
        reader, content_length = data, get_content_length(data)
    resp = _blob_create_response  # set when _blob_upload_bytes already made the request
    if resp is None:
        resp = await stub.BlobCreate(
            BlobCreateRequest(
                content_md5=upload_hashes.md5_base64,
                content_sha256_base64=upload_hashes.sha256_base64,
                content_length=content_length,
            )
        )
    if resp.WhichOneof("upload_types_oneof") == "multiparts":
        if reader is None:
            reader = BytesIO(data)

        async def send_multipart(part):
            return await perform_multipart_upload(
                reader,
                content_length=content_length,
                max_part_size=part.part_length,
                part_urls=part.upload_urls,
                completion_url=part.completion_url,
                upload_chunk_size=DEFAULT_SEGMENT_CHUNK_SIZE,
                progress_report_cb=progress_report_cb,
                byte_budget=byte_budget,
            )

        result = await _blob_upload_with_fallback(resp.multiparts.items, resp.blob_ids, send_multipart, content_length)
    else:
        payload = None

        async def send_single(url):
            nonlocal payload
            if payload is None:
                # the whole-blob MD5 is already in upload_hashes: hand it to the payload instead of re-hashing
                raw = getattr(upload_hashes, "md5_raw", None)
                if raw is None and _is_real_md5(upload_hashes):
                    raw = bytes.fromhex(upload_hashes.md5_hex())
                if reader is None and raw is not None:
                    payload = KnownBytesBody(data, raw, progress_report_cb)  # in memory, digest known: no reader at all
                else:
                    payload = BytesIOSegmentPayload(
                        reader if reader is not None else BytesIO(data), segment_start=0, segment_length=content_length,
                        progress_report_cb=progress_report_cb, md5_digest=raw)
            return await _upload_to_s3_url(url, payload, content_md5_b64=upload_hashes.md5_base64)

        result = await _blob_upload_with_fallback(resp.upload_urls.items, resp.blob_ids, send_single, content_length)
    if progress_report_cb:
        progress_report_cb(complete=True)
    return result


async def _blob_upload_bytes(upload_hashes: UploadHashes, data: bytes, stub) -> tuple[str, bool, int]:
    """``_blob_upload`` for an in-memory payload whose digests came out of a GPU batch (see ``_blob_upload_row``)."""
    return await _blob_upload_row(upload_hashes.md5_base64, upload_hashes.sha256_base64,
                                  getattr(upload_hashes, "md5_raw", None), data, stub)


async def _blob_upload_row(md5_b64: str, sha256_b64: str, md5_raw: bytes | None, data: bytes, stub) -> tuple[str, bool, int]:
    """``_blob_upload`` for the map pump's case -- an in-memory payload and its row of a GPU digest table (base64
    columns + the raw MD5) -- with the single-PUT branch and the provider fallback written out flat (same BlobCreate
    request, same fallback order, same r2 bookkeeping as ``_blob_upload`` / ``_blob_upload_with_fallback``): 10^5 of
    these run per map on the event-loop thread, and every coroutine frame, closure and temporary object per input is
    paid there.  Anything else (multipart answer, digest unknown) goes through the general function."""
    resp = await stub.BlobCreate(BlobCreateRequest(content_md5=md5_b64, content_sha256_base64=sha256_b64,
                                                   content_length=len(data)))  # keywords: the real class is a protobuf
    if md5_raw is None or resp.WhichOneof("upload_types_oneof") != "upload_urls":
        return await _blob_upload(hash_utils._UploadHashesRaw(md5_b64, sha256_b64, md5_raw), data, stub,
                                  _blob_create_response=resp)
    body = KnownBytesBody(data, md5_raw)
    urls, blob_ids = resp.upload_urls.items, resp.blob_ids
    if len(urls) == 1 and not blob_ids[0].endswith(":r2"):  # the common answer: one provider, nothing to fall back to
        await _upload_to_s3_url(urls[0], body, content_md5_b64=md5_b64)
        return blob_ids[0], False, 0
    r2_failed, last = False, len(urls) - 1
    for idx, url in enumerate(urls):
        blob_id = blob_ids[idx]
        is_r2 = blob_id.endswith(":r2")
        try:
            if is_r2:
                t0 = time.monotonic_ns()
                await _upload_to_s3_url(url, body, content_md5_b64=md5_b64)
                return blob_id, r2_failed, (len(data) * 1_000_000_000) // max(time.monotonic_ns() - t0, 1)
            await _upload_to_s3_url(url, body, content_md5_b64=md5_b64)
            return blob_id, r2_failed, 0
        except Exception:
            r2_failed = r2_failed or is_r2
            if idx == last:
                raise
    raise ExecutionError("Failed to upload blob")


def _is_real_md5(h: UploadHashes) -> bool:
    return bool(h.md5_base64) and h.md5_hex() != _MD5_PLACEHOLDER


def _is_real_md5_hex(md5_hex: str | None) -> bool:
    return bool(md5_hex) and md5_hex != _MD5_PLACEHOLDER


async def blob_upload_with_r2_failure_info(payload: bytes, stub) -> tuple[str, bool, int]:
    if isinstance(payload, str):
        logger.debug("Blob uploading string, not bytes - auto-encoding as utf8")
        payload = payload.encode("utf8")
    t0 = time.time()
    hashes = get_upload_hashes(payload)
    out = await _blob_upload(hashes, payload, stub)
    mib = len(payload) / (1 << 20)
    dt = max(time.time() - t0, 0.001)
    logger.debug(f"Uploaded large blob of size {mib:.2f} MiB ({mib / dt:.2f} MiB/s, total {dt:.2f}s). {out[0]}")
    return out


async def blob_upload(payload: bytes, stub) -> str:
    blob_id, _, _ = await blob_upload_with_r2_failure_info(payload, stub)
    return blob_id


async def blob_upload_many(payloads: Sequence[bytes], stub, concurrency: int | None = None) -> list[tuple[str, bool, int]]:
    """The batched form the map pump uses: hash all payloads in ONE GPU batch, then run the uploads with
    the reference's concurrency (BLOB_MAX_PARALLELISM).  Order is preserved."""
    payloads = [p.encode("utf8") if isinstance(p, str) else p for p in payloads]
    hashes = await asyncio.to_thread(hash_utils.get_upload_hashes_many, payloads)
    jobs = list(zip(hashes, payloads))
    return await bounded_map(jobs, lambda hp: _blob_upload(hp[0], hp[1], stub), concurrency or BLOB_MAX_PARALLELISM)


async def format_blob_data(data: bytes, api_stub) -> dict[str, Any]:
    return {"data_blob_id": await blob_upload(data, api_stub)} if len(data) > MAX_OBJECT_SIZE_BYTES else {"data": data}


async def blob_upload_file(
    file_obj: BinaryIO,
    stub,
    progress_report_cb: Callable | None = None,
    sha256_hex: str | None = None,
    md5_hex: str | None = None,
    byte_budget: _ByteBudget | None = None,
) -> str:
    hashes = get_upload_hashes(file_obj, sha256_hex=sha256_hex, md5_hex=md5_hex)
    blob_id, _, _ = await _blob_upload(hashes, file_obj, stub, progress_report_cb, byte_budget=byte_budget)
    return blob_id


# ------------------------------------------------------------------------------------------- download


@retry(n_attempts=5, base_delay=0.1, attempt_timeout=None)
async def _download_from_url(download_url: str) -> bytes:
    """GET one blob (reference :377-388; no integrity check there either: blobs are addressed by id)."""
    async with ClientSessionRegistry.get_session().get(download_url) as s3_resp:
        if s3_resp.status == 503:  # S3 SlowDown
            logger.debug("Received SlowDown signal from S3, sleeping for 1 second before retrying.")
            await asyncio.sleep(1)
        if s3_resp.status != 200:
            text = await s3_resp.text()
            raise ExecutionError(f"Get from url failed with status {s3_resp.status}: {text}")
        return await s3_resp.read()


async def blob_download(blob_id: str, stub) -> bytes:
    """Read a whole blob into memory (reference :391-404)."""
    logger.debug(f"Downloading large blob {blob_id}")
    t0 = time.time()
    resp = await stub.BlobGet(_wire.BlobGetRequest(blob_id=blob_id))
    data = await _download_from_url(resp.download_url)
    size_mib = len(data) / 1024 / 1024
    dur_s = max(time.time() - t0, 0.001)
    logger.debug(f"Downloaded large blob {blob_id} of size {size_mib:.2f} MiB ({size_mib / dur_s:.2f} MiB/s, total {dur_s:.2f}s)")
    return data


async def blob_iter(blob_id: str, stub):
    """Stream a blob chunk by chunk (reference :407-422)."""
    resp = await stub.BlobGet(_wire.BlobGetRequest(blob_id=blob_id))
    async with ClientSessionRegistry.get_session().get(resp.download_url) as s3_resp:
        if s3_resp.status == 503:
            logger.debug("Received SlowDown signal from S3, sleeping for 1 second before retrying.")
            await asyncio.sleep(1)
        if s3_resp.status != 200:
            text = await s3_resp.text()
            raise ExecutionError(f"Get from url failed with status {s3_resp.status}: {text}")
        async for chunk in s3_resp.content.iter_any():
            yield chunk


# ------------------------------------------------------------------------------- FileUploadSpec (v1)


@dataclasses.dataclass(slots=True)
class FileUploadSpec:
    source: Callable[[], AbstractContextManager | BinaryIO]
    source_description: Any
    source_is_path: bool
    mount_filename: str

    use_blob: bool
    sha256_hex: str
    md5_hex: str
    mode: int  # permission bits (low 12 bits of st_mode)
    size: int
    content: bytes | None = None  # cached for very small files

    def read_content(self) -> bytes:
        with self.source() as fp:
            fp.seek(0)
            return fp.read()


def _size_class(size: int) -> tuple[bool, bool, bool]:
    """-> (use_blob, want_md5, cache_content) for a file of ``size`` bytes (reference :459-474)."""
    if size >= LARGE_FILE_LIMIT:
        return True, not (size > MULTIPART_UPLOAD_THRESHOLD), False
    return False, True, size < SMALL_FILE_INLINE_LIMIT


def _get_file_upload_spec(
    source: Callable[[], AbstractContextManager | BinaryIO],
    source_description: Any,
    mount_filename: PurePosixPath,
    mode: int,
) -> FileUploadSpec:
    content = None
    with source() as fp:
        size = fp.seek(0, os.SEEK_END)  # the current position is ignored: uploads start at 0
        fp.seek(0)
        use_blob, want_md5, cache = _size_class(size)
        if cache:
            content = fp.read()
            hashes = get_upload_hashes(content)
        else:
            hashes = get_upload_hashes(fp, md5_hex=None if want_md5 else _MD5_PLACEHOLDER)
    return FileUploadSpec(
        source=source,
        source_description=source_description,
        source_is_path=isinstance(source_description, Path),
        mount_filename=mount_filename.as_posix(),
        use_blob=use_blob,
        sha256_hex=hashes.sha256_hex(),
        md5_hex=hashes.md5_hex(),
        mode=mode & 0o7777,
        size=size,
        content=content,
    )


def _default_mode(filename: Path) -> int:
    return os.stat(filename).st_mode & (0o7777 if platform.system() != "Windows" else 0o7755)


def get_file_upload_spec_from_path(
    filename: Path, mount_filename: PurePosixPath, mode: int | None = None
) -> FileUploadSpec:
    return _get_file_upload_spec(lambda: open(filename, "rb"), filename, mount_filename, mode or _default_mode(filename))


def get_file_upload_spec_from_fileobj(fp: BinaryIO, mount_filename: PurePosixPath, mode: int) -> FileUploadSpec:
    @contextmanager
    def source():
        fp.seek(0)
        yield fp

    return _get_file_upload_spec(source, str(fp), mount_filename, mode)


def get_file_upload_specs(
    files: Sequence[tuple[Path | str, PurePosixPath | str, int | None]],
    cache_small_content: bool | None = None,
) -> list[FileUploadSpec]:
    """Batched ``get_file_upload_spec_from_path``: every file of a ``Volume.batch_upload`` / ``Mount`` goes
    to the GPU in one batch (the reference fans the per-file hashlib loops over a ThreadPoolExecutor,
    py/modal/volume.py:1209-1216, py/modal/mount.py:467-485).  Sizes/modes come from ``b200h_stat_files`` and
    the bytes are read by the library's native reader threads straight into its pinned staging ring
    (``b200h_hash_files``): no per-file Python I/O, no mmap.
    Same size classes / placeholder MD5 as ``_get_file_upload_spec``.  ``content`` (the reference's
    "avoid the double read" cache for files < 256 KiB) is filled when ``cache_small_content`` is true;
    the default (None) does so only for batches of <= 4096 files -- for a million-file tree the extra
    Python read per file would cost more than the hashing."""
    if not files:
        return []
    ctx = get_context()
    n = len(files)
    paths = [os.fsencode(f[0]) for f in files]  # encoded once for the stat and the hash calls
    sizes, modes = ctx.stat_files(paths)
    # size classes, vectorised (same comparisons as _size_class)
    use_blob = sizes >= LARGE_FILE_LIMIT
    want_md5 = ~(use_blob & (sizes > MULTIPART_UPLOAD_THRESHOLD))
    cacheable = ~use_blob & (sizes < SMALL_FILE_INLINE_LIMIT)
    if cache_small_content is None:
        cache_small_content = n <= 4096
    # Files whose content is cached in the spec (< 256 KiB, like the reference's "read once" class) are read ONCE, here,
    # and those very bytes are hashed -- the digest can never disagree with spec.content, whatever happens to the
    # file meanwhile.  Everything else is read by the library's native reader.
    contents: dict[int, bytes] = {}
    if cache_small_content:
        for i in np.flatnonzero(cacheable).tolist():
            with open(files[i][0], "rb") as f:
                contents[i] = f.read()
        if contents:
            idx = np.fromiter(contents.keys(), dtype=np.int64, count=len(contents))
            sizes[idx] = [len(c) for c in contents.values()]
    from_memory = np.zeros(n, bool)
    if contents:
        from_memory[list(contents.keys())] = True
    # one fused SHA-256+MD5 batch for the files that need both, a SHA-only batch for the > 1 GiB class.  The digest
    # columns come back as the hex text the wire rows carry (FileUploadSpec / MountFile.sha256_hex), formatted on the
    # device from the digest table (B200H_HEX_OUT) -- no per-row conversion on the host.
    HEX = _lib.HEX_OUT
    sha_all = np.empty((n, 64), np.uint8)
    md5_all = np.full((n, 32), ord("0"), np.uint8)
    if contents:
        idx = np.flatnonzero(from_memory)
        sha, md5, _ = ctx.hash_buffers([contents[i] for i in idx.tolist()], _lib.SHA256 | _lib.MD5 | HEX)
        sha_all[idx], md5_all[idx] = sha, md5
    both = np.flatnonzero(want_md5 & ~from_memory)
    sha_only = np.flatnonzero(~want_md5 & ~from_memory)
    if both.size:
        sha, md5, _ = ctx.hash_files([paths[i] for i in both] if both.size != n else paths, sizes[both], 0,
                                     _lib.SHA256 | _lib.MD5 | HEX)
        sha_all[both], md5_all[both] = sha, md5
    if sha_only.size:
        sha, _, _ = ctx.hash_files([paths[i] for i in sha_only], sizes[sha_only], 0, _lib.SHA256 | HEX)
        sha_all[sha_only] = sha
    # A file that GREW between the stat and the read was hashed as its old prefix (a file that shrank fails the read):
    # stat again and redo the few that changed one at a time, the reference's way (one open, size and bytes together).
    redo: dict[int, FileUploadSpec] = {}
    streamed = np.flatnonzero(~from_memory)
    if streamed.size:
        sizes_after, _ = ctx.stat_files([paths[i] for i in streamed] if streamed.size != n else paths)
        for i in streamed[sizes_after != sizes[streamed]].tolist():
            filename, mount_filename, mode = files[i]
            redo[i] = get_file_upload_spec_from_path(Path(filename), PurePosixPath(mount_filename), mode)
    sha_hex, md5_hex = sha_all.tobytes().decode("ascii"), md5_all.tobytes().decode("ascii")  # sliced per file below
    sizes_l, modes_l = sizes.tolist(), modes.tolist()
    use_blob_l, want_md5_l = use_blob.tolist(), want_md5.tolist()
    # The per-file Python work below is what is left of a million-file tree once hashing takes a fraction of a second,
    # so it is kept to positional construction and precomputed columns (~2.5 us per file).
    partial, spec_cls, placeholder = functools.partial, FileUploadSpec, _MD5_PLACEHOLDER
    specs = []
    append = specs.append
    # a million small objects allocated in one go: without this the cyclic GC rescans the growing list again and again
    gc_was_on = gc.isenabled()
    gc.disable()
    try:
        _build_specs(files, append, spec_cls, partial, placeholder, contents, use_blob_l, want_md5_l,
                     sha_hex, md5_hex, modes_l, sizes_l)
    finally:
        if gc_was_on:
            gc.enable()
    for i, spec in redo.items():
        specs[i] = spec
    return specs


def _build_specs(files, append, spec_cls, partial, placeholder, contents, use_blob_l, want_md5_l,
                 sha_hex, md5_hex, modes_l, sizes_l) -> None:
    get_content = contents.get
    for i, (filename, mount_filename, mode) in enumerate(files):
        content = get_content(i)  # the bytes that were hashed (cached class only)
        append(
            spec_cls(
                partial(open, filename, "rb"),                                        # source
                filename if isinstance(filename, Path) else Path(filename),           # source_description
                True,                                                                 # source_is_path
                mount_filename if type(mount_filename) is str                         # posix string from a trusted walk
                else str(mount_filename) if type(mount_filename) is PurePosixPath
                else PurePosixPath(mount_filename).as_posix(),
                use_blob_l[i],
                sha_hex[64 * i : 64 * i + 64],
                md5_hex[32 * i : 32 * i + 32] if want_md5_l[i] else placeholder,
                (mode if mode else modes_l[i]) & 0o7777,
                sizes_l[i],
                content,
            )
        )


def first_occurrence_of_specs(specs: Sequence[FileUploadSpec]) -> tuple[list[int], int]:
    """In-batch dedupe of a list of specs by content (SHA-256), computed on the GPU over the digest table:
    ``first[i]`` is the index of the first spec with the same content as spec i.  The reference's counterpart is
    the ``accounted_hashes`` set walked file by file in ``_Mount._load_mount`` (py/modal/mount.py:498,518-534)."""
    n = len(specs)
    if n == 0:
        return [], 0
    keys = np.frombuffer(bytes.fromhex("".join(s.sha256_hex for s in specs)), np.uint8).reshape(n, 32)
    first, ndistinct = get_context().dedupe(keys)
    return first.tolist(), ndistinct


# ---------------------------------------------------------------------------- FileUploadSpec2 (v2)

_FileUploadSource2 = Callable[[], ContextManager[BinaryIO]]


@dataclasses.dataclass
class FileUploadBlock:
    start: int  # inclusive byte offset of the block in the file
    end: int  # exclusive end after dropping the block's trailing zero bytes
    contents_sha256: bytes  # raw 32-byte SHA-256 of [start, end)


def _blocks_of(view: np.ndarray) -> list[FileUploadBlock]:
    """All ceil(size/BLOCK_SIZE) blocks of one file image: trim scan + SHA-256 per block on the device."""
    if view.size == 0:
        return []
    sha, _, trimmed, _ = get_context().hash_fixed_parts(view, BLOCK_SIZE, _lib.SHA256 | _lib.TRIM_ZEROS)
    return _blocks_from_table(sha, trimmed)


def _blocks_of_device(fp: DeviceFile) -> list[FileUploadBlock]:
    """The same blocks of a buffer in GPU memory, trimmed and hashed where it is: only the (trimmed length, SHA-256)
    table crosses to the host."""
    sha, _, trimmed = fp.hash_parts(BLOCK_SIZE, _lib.SHA256 | _lib.TRIM_ZEROS)
    return _blocks_from_table(sha, trimmed)


def _blocks_from_table(sha: np.ndarray, trimmed: np.ndarray) -> list[FileUploadBlock]:
    return [
        FileUploadBlock(start=i * BLOCK_SIZE, end=i * BLOCK_SIZE + int(trimmed[i]), contents_sha256=sha[i].tobytes())
        for i in range(len(trimmed))
    ]


@dataclasses.dataclass
class FileUploadSpec2:
    source: _FileUploadSource2
    source_description: str | Path

    path: str
    blocks: list[FileUploadBlock]  # 8 MiB blocks
    mode: int
    size: int

    @staticmethod
    async def from_path(
        filename: Path, mount_filename: PurePosixPath, hash_semaphore: asyncio.Semaphore, mode: int | None = None
    ) -> "FileUploadSpec2":
        def source():
            return open(filename, "rb")

        return await FileUploadSpec2._create(source, filename, mount_filename, mode or _default_mode(filename),
                                             hash_semaphore)

    @staticmethod
    async def from_fileobj(
        source_fp: BinaryIO | BytesIO | DeviceFile, mount_filename: PurePosixPath, hash_semaphore: asyncio.Semaphore,
        mode: int
    ) -> "FileUploadSpec2":
        if isinstance(source_fp, DeviceFile):
            # every use gets its own reader over the same device bytes (the missing-block PUTs run concurrently)
            return await FileUploadSpec2._create(source_fp.reopen, repr(source_fp), mount_filename, mode, hash_semaphore)
        try:
            fileno = source_fp.fileno()

            def source():
                fp = os.fdopen(os.dup(fileno), "rb")
                fp.seek(0)
                return fp

        except OSError:  # BytesIO-like: no descriptor
            buffer = source_fp.getbuffer()

            def source():
                return BytesIO(buffer)

        return await FileUploadSpec2._create(source, str(source), mount_filename, mode, hash_semaphore)

    @staticmethod
    async def _create(
        source: _FileUploadSource2,
        source_description: str | Path,
        mount_filename: PurePosixPath,
        mode: int,
        hash_semaphore: asyncio.Semaphore,
    ) -> "FileUploadSpec2":
        with source() as fp:
            size = fp.seek(0, os.SEEK_END)
        blocks = await _gather_blocks(source, size, hash_semaphore)
        return FileUploadSpec2(source=source, source_description=source_description, path=mount_filename.as_posix(),
                               blocks=blocks, mode=mode & 0o7777, size=size)


async def _gather_blocks(source: _FileUploadSource2, size: int, hash_semaphore: asyncio.Semaphore) -> list[FileUploadBlock]:
    """Block list of one file.  The reference launches one thread task per block, each reading its block
    twice (rstrip pass + SHA pass, :640-664); here the file image is handed to the GPU once and all its
    blocks are trimmed and hashed by one batch."""
    if size == 0:
        return []

    def run() -> list[FileUploadBlock]:
        with source() as fp:
            if isinstance(fp, DeviceFile):
                return _blocks_of_device(fp)
            return _with_view(fp, lambda view: _blocks_of(view[:size]))

    async with hash_semaphore:
        return await asyncio.to_thread(run)


def _read_range(source: _FileUploadSource2, start: int, end: int) -> bytes:
    with source() as fp:
        fp.seek(start)
        out = bytearray()
        while len(out) < end - start:
            chunk = fp.read(end - start - len(out))
            if not chunk:
                break
            out += chunk
        return bytes(out)


def _gather_block(source: _FileUploadSource2, block_idx: int) -> FileUploadBlock:
    start = block_idx * BLOCK_SIZE
    data = _read_range(source, start, start + BLOCK_SIZE)
    sha, _, trimmed = get_context().hash_batch_host(np.frombuffer(data, dtype=np.uint8), [0], [len(data)],
                                                    _lib.SHA256 | _lib.TRIM_ZEROS)
    return FileUploadBlock(start=start, end=start + int(trimmed[0]), contents_sha256=sha[0].tobytes())


def _hash_range_sha256(source: _FileUploadSource2, start, end) -> bytes:
    data = _read_range(source, start, end)
    sha, _, _ = get_context().hash_buffers([data], _lib.SHA256)
    return sha[0].tobytes()


def _find_end_of_block(source: _FileUploadSource2, start: int, end: int) -> int | None:
    """Index just past the last non-zero byte of [start, end) -- ``start`` for an empty or all-zero range.
    (The reference docstring's ``(…, 0, 3) -> 4`` example is stale: its code, like this, returns 3.)"""
    data = _read_range(source, start, end)
    if not data:
        return start
    _, _, trimmed = get_context().hash_batch_host(np.frombuffer(data, dtype=np.uint8), [0], [len(data)],
                                                  _lib.SHA256 | _lib.TRIM_ZEROS)
    return start + int(trimmed[0])


async def file_upload_specs2(
    files: Sequence[tuple[Path, PurePosixPath, int | None]],
) -> list[FileUploadSpec2]:
    """Batched ``FileUploadSpec2.from_path`` for a whole ``batch_upload``: the blocks of ALL files form one
    GPU batch (so a tree of many small files is as efficient as one big file), read by the library's native
    reader threads (``b200h_hash_files`` with part_len = BLOCK_SIZE and zero trimming)."""
    if not files:
        return []

    def run() -> list[FileUploadSpec2]:
        ctx = get_context()
        paths = [os.fsencode(f[0]) for f in files]  # encoded once for the stat and the hash calls
        sizes, modes = ctx.stat_files(paths)
        sha, _, trimmed = ctx.hash_files(paths, sizes, BLOCK_SIZE, _lib.SHA256 | _lib.TRIM_ZEROS)
        out, row = [], 0
        sizes_l, modes_l, trimmed_l, sha_raw = sizes.tolist(), modes.tolist(), trimmed.tolist(), sha.tobytes()
        block_cls, spec_cls, partial, bs = FileUploadBlock, FileUploadSpec2, functools.partial, BLOCK_SIZE
        gc_was_on = gc.isenabled()
        gc.disable()  # bulk allocation of small objects: keep the cyclic GC from rescanning the growing lists
        try:
            for i, (filename, mount_filename, mode) in enumerate(files):
                size = sizes_l[i]
                blocks = []
                for start in range(0, size, bs):
                    blocks.append(block_cls(start, start + trimmed_l[row], sha_raw[32 * row : 32 * row + 32]))
                    row += 1
                out.append(
                    spec_cls(
                        source=partial(open, filename, "rb"),
                        source_description=filename if isinstance(filename, Path) else Path(filename),
                        path=mount_filename if type(mount_filename) is str
                        else str(mount_filename) if type(mount_filename) is PurePosixPath
                        else PurePosixPath(mount_filename).as_posix(),
                        blocks=blocks,
                        mode=(mode if mode else modes_l[i]) & 0o7777,
                        size=size,
                    )
                )
        finally:
            if gc_was_on:
                gc.enable()
        return out

    return await asyncio.to_thread(run)


async def device_file_specs2(
    items: Sequence[tuple[DeviceFile, PurePosixPath, int]],
) -> list[FileUploadSpec2]:
    """Batched ``FileUploadSpec2.from_fileobj`` for the ``DeviceFile``s of one ``batch_upload``: the blocks of ALL of
    them, whatever tensors they are made of, are trimmed and hashed by one ``b200h_hash_segment_parts_device`` call,
    and only that table comes to the host."""
    if not items:
        return []

    def run() -> list[FileUploadSpec2]:
        files = [fp for fp, _, _ in items]
        sha, _, trimmed = hash_parts_many(files, BLOCK_SIZE, _lib.SHA256 | _lib.TRIM_ZEROS, ctx=get_context())
        out, row = [], 0
        for fp, remote, mode in items:
            n = -(-fp.nbytes // BLOCK_SIZE)
            out.append(FileUploadSpec2(source=fp.reopen, source_description=repr(fp),
                                       path=PurePosixPath(remote).as_posix(),
                                       blocks=_blocks_from_table(sha[row : row + n], trimmed[row : row + n]),
                                       mode=mode & 0o7777, size=fp.nbytes))
            row += n
        return out

    return await asyncio.to_thread(run)


def use_md5(url: str) -> bool:
    """Attach Content-MD5 only for real S3 / R2 hosts (moto and local fakes reject it; reference :708-727)."""
    host = urlparse(url).netloc.split(":")[0]
    if host.endswith((".amazonaws.com", ".r2.cloudflarestorage.com")):
        return True
    if host == "localhost":
        return False
    try:
        import ipaddress

        addr = ipaddress.ip_address(host)
        if addr.is_private or addr.is_loopback:
            return False
    except ValueError:
        pass
    raise Exception(f"Unknown S3 host: {host}")
