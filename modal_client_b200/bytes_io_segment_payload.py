"""aiohttp payload that streams one segment of a file and knows that segment's MD5.

Counterpart of the reference's ``BytesIOSegmentPayload`` (py/modal/_utils/bytes_io_segment_payload.py:19-116):
same constructor, attributes and methods, because ``_upload_to_s3_url`` / ``perform_multipart_upload`` /
``_put_missing_blocks`` drive it through exactly that surface.  What differs is where the digest comes from.
The reference folds every chunk it sends into a ``hashlib.md5`` on an executor thread, i.e. it hashes every
uploaded byte a second time on the CPU.  Here the segment MD5 normally arrives *precomputed* from the GPU batch
that hashed all parts at once (``md5_digest=``), so sending is a pure read+write loop; only when no digest was
supplied are the chunks folded into a device-resident ``DigestStream`` (``b200h_stream_*``), which offers the
``update`` / ``hexdigest`` shape the callers expect from the hashlib object.
"""
from __future__ import annotations

import asyncio
import contextlib
from collections.abc import Callable
from typing import BinaryIO

from aiohttp import BytesPayload, Payload
from aiohttp.abc import AbstractStreamWriter

from ._backend import get_context
from ._lib import MD5

DEFAULT_SEGMENT_CHUNK_SIZE = 1 << 24  # 16 MiB per read


class _DigestKnown:
    """hashlib-shaped view of a digest the GPU batch already produced."""

    __slots__ = ("_raw",)

    def __init__(self, raw: bytes):
        self._raw = raw

    def update(self, _chunk) -> None:
        pass  # nothing to fold: the bytes were hashed before the upload started

    def digest(self) -> bytes:
        return self._raw

    def hexdigest(self) -> str:
        return self._raw.hex()


class _DigestOnDevice:
    """hashlib-shaped incremental MD5 whose chaining state lives on the GPU."""

    def __init__(self):
        self._stream = None  # created on first use: most payloads are reset without ever being hashed

    def _dev(self):
        if self._stream is None:
            self._stream = get_context().stream(MD5)
        return self._stream

    def update(self, chunk) -> None:
        self._dev().update(chunk)

    def digest(self) -> bytes:
        return self._dev().digests()[1]

    def hexdigest(self) -> str:
        return self.digest().hex()

    def close(self) -> None:
        if self._stream is not None:
            self._stream.close()
            self._stream = None


def _ignore_progress(*_args, **_kwargs):
    return None


class BytesIOSegmentPayload(Payload):
    """Body of one PUT: bytes ``[segment_start, segment_start + segment_length)`` of ``bytes_io`` counted from
    the position the reader had when the payload was built.  The reader must not be shared (its position is
    moved without locking)."""

    _value: BinaryIO

    def __init__(
        self,
        bytes_io: BinaryIO,
        segment_start: int,
        segment_length: int,
        chunk_size: int = DEFAULT_SEGMENT_CHUNK_SIZE,
        progress_report_cb: Callable | None = None,
        md5_digest: bytes | None = None,  # raw 16 bytes when the GPU batch already produced it
    ):
        super().__init__(bytes_io)
        self.initial_seek_pos = bytes_io.tell()
        self.segment_start, self.segment_length = segment_start, segment_length
        self.chunk_size = chunk_size
        self.progress_report_cb = progress_report_cb if progress_report_cb is not None else _ignore_progress
        self._size = segment_length
        self._given_digest = md5_digest
        self._md5_checksum = None
        # aiohttp's size probe looks from the current position: park the reader at the segment start for it
        bytes_io.seek(self.initial_seek_pos + segment_start)
        if segment_length > super().size:
            raise AssertionError("segment reaches past the end of the stream")
        self.reset_state()

    # ---- state -------------------------------------------------------------------------------------------
    def reset_state(self):
        """Back to 'nothing sent': a retry re-reads (and, without a given digest, re-hashes) from scratch."""
        previous = self._md5_checksum
        if isinstance(previous, _DigestOnDevice):
            previous.close()
        self._md5_checksum = _DigestOnDevice() if self._given_digest is None else _DigestKnown(self._given_digest)
        self.num_bytes_read = 0
        self._value.seek(self.initial_seek_pos)

    @contextlib.contextmanager
    def reset_on_error(self, subtract_progress: bool = False):
        failed = None
        try:
            yield
        except Exception as exc:  # report the lost progress, then let the caller's retry logic see the error
            failed = exc
        finally:
            sent = self.num_bytes_read
            self.reset_state()
        if failed is not None:
            try:
                if subtract_progress:
                    self.progress_report_cb(advance=-sent)
                else:
                    self.progress_report_cb(reset=True)
            except Exception as cb_exc:
                raise cb_exc from failed
            raise failed

    # ---- what aiohttp and the upload functions ask ---------------------------------------------------------
    @property
    def size(self) -> int:
        return self.segment_length

    def md5_checksum(self):
        return self._md5_checksum

    def remaining_bytes(self) -> int:
        return self.segment_length - self.num_bytes_read

    def decode(self, encoding: str = "utf-8", errors: str = "strict") -> str:
        self._value.seek(self.initial_seek_pos)
        return self._value.read().decode(encoding, errors)

    async def write(self, writer: "AbstractStreamWriter"):
        await self.write_with_length(writer, None)  # aiohttp < 3.12 enters here

    async def write_with_length(self, writer: AbstractStreamWriter, content_length: int | None):
        loop = asyncio.get_event_loop()
        limit = self.segment_length if content_length is None else min(self.segment_length, content_length)
        origin = self.initial_seek_pos + self.segment_start
        while self.num_bytes_read < limit:
            self._value.seek(origin + self.num_bytes_read)
            chunk = await loop.run_in_executor(None, self._value.read, min(self.chunk_size, limit - self.num_bytes_read))
            if not chunk:
                break  # stream ended early; the ETag comparison will flag it
            if self._given_digest is None:
                await loop.run_in_executor(None, self._md5_checksum.update, chunk)
            self.num_bytes_read += len(chunk)
            await writer.write(chunk)
            self.progress_report_cb(advance=len(chunk))


class MemorySegmentPayload(BytesPayload):
    """Body of one PUT whose bytes already lie in host memory (a ``memoryview`` into a staging buffer): sent from
    where they are, ``chunk_size`` bytes per write with the progress reports and the ``reset_on_error`` behaviour of
    ``BytesIOSegmentPayload``, without reading, copying or hashing anything."""

    def __init__(self, data: memoryview, chunk_size: int = DEFAULT_SEGMENT_CHUNK_SIZE,
                 progress_report_cb: Callable | None = None):
        super().__init__(data)
        self.chunk_size = chunk_size
        self.progress_report_cb = progress_report_cb if progress_report_cb is not None else _ignore_progress
        self.num_bytes_read = 0

    @contextlib.contextmanager
    def reset_on_error(self, subtract_progress: bool = False):
        try:
            yield
        except Exception as failed:
            sent, self.num_bytes_read = self.num_bytes_read, 0
            try:
                if subtract_progress:
                    self.progress_report_cb(advance=-sent)
                else:
                    self.progress_report_cb(reset=True)
            except Exception as cb_exc:
                raise cb_exc from failed
            raise
        self.num_bytes_read = 0

    async def write(self, writer: AbstractStreamWriter):
        await self.write_with_length(writer, None)  # aiohttp < 3.12 enters here

    async def write_with_length(self, writer: AbstractStreamWriter, content_length: int | None):
        limit = len(self._value) if content_length is None else min(len(self._value), content_length)
        while self.num_bytes_read < limit:
            chunk = self._value[self.num_bytes_read : min(limit, self.num_bytes_read + self.chunk_size)]
            await writer.write(chunk)
            self.num_bytes_read += len(chunk)
            self.progress_report_cb(advance=len(chunk))


class KnownBytesBody:
    """An in-memory blob on its way to a single-part PUT together with the MD5 the GPU batch already produced for it.
    The map pump creates one per blobified input (10^5 per map), so this is a two-slot record; the aiohttp payload
    is only built by ``as_payload()`` when a PUT really goes out.  The reference wraps every blob in a BytesIO and a
    BytesIOSegmentPayload, whose ``write`` then hops to an executor thread per 16 MiB chunk to read memory that is
    already in memory and to re-hash it (bytes_io_segment_payload.py:96-106)."""

    __slots__ = ("data", "md5_raw", "progress_report_cb")

    def __init__(self, data: bytes, md5_raw: bytes, progress_report_cb: Callable | None = None):
        self.data, self.md5_raw, self.progress_report_cb = data, md5_raw, progress_report_cb

    @property
    def size(self) -> int:
        return len(self.data)

    def md5_checksum(self) -> _DigestKnown:
        return _DigestKnown(self.md5_raw)

    @contextlib.contextmanager
    def reset_on_error(self, subtract_progress: bool = False):
        try:
            yield  # nothing to rewind: the body is immutable bytes, the digest is final
        except Exception:
            if self.progress_report_cb is not None:
                self.progress_report_cb(advance=-len(self.data)) if subtract_progress else self.progress_report_cb(reset=True)
            raise

    def as_payload(self) -> "Payload":
        body = _ReportingBytesPayload(self.data)
        body.progress_report_cb = self.progress_report_cb
        return body


class _ReportingBytesPayload(BytesPayload):
    progress_report_cb: Callable | None = None

    async def write(self, writer: AbstractStreamWriter):
        await super().write(writer)
        if self.progress_report_cb is not None:
            self.progress_report_cb(advance=len(self._value))
