"""A read-only file object over bytes that live in GPU memory: one CUDA tensor, or a safetensors image of many.

``DeviceFile(t)`` lets a buffer that lives in GPU memory -- a checkpoint shard, a safetensors image, an embedding
table -- go wherever the upload functions accept a ``BinaryIO``, without first copying the whole buffer to host memory.
``DeviceFile.safetensors(state_dict)`` is the same for a whole checkpoint: a file whose bytes are exactly what
``safetensors.torch.save(state_dict)`` would produce, made of the tensors where they are (plus a small header), so the
image is never assembled, neither in host memory nor in HBM.

* volumefs2 (``VolumeUploadContextManager2.put_file`` / ``FileUploadSpec2.from_fileobj``) recognises it and trims and
  hashes its 8 MiB blocks in place (``hash_parts``): one tensor with one ``b200h_hash_fixed_parts_device`` call, a
  file made of several tensors with one ``b200h_hash_segment_parts_device`` call, which gathers only the blocks that
  straddle tensor boundaries.  Only the (trimmed length, SHA-256) table comes to the host, and afterwards only the
  trimmed bytes of the blocks the server reports missing are read.
* every other consumer (volumefs1 ``put_file``, ``get_file_upload_spec_from_fileobj``, ``blob_upload_file``) reads it
  like any other stream.  Those digests are one serial chain over the whole object and gain nothing from the GPU.

``read`` / ``readinto`` copy device -> host through one page-locked bounce buffer of bounded size (16 MiB by default),
so host memory never has to hold the tensors.  ``bytes_to_host`` counts what has crossed.  The readers ``reopen()``
hands out share the tensors, the bounce buffer and that counter.  The tensors must not change while an upload reads
them.
"""
from __future__ import annotations

import bisect
import io
import json
import os
import threading
from collections.abc import Mapping

import numpy as np

from . import _lib
from ._backend import get_context

BOUNCE_BYTES = 16 << 20  # page-locked host memory per DeviceFile (shared by its reopen() readers)


class _TensorBytes:
    """The bytes of an ordered list of contiguous CUDA tensors (the segments), read as one file, plus what reading them
    needs: a side stream ordered after the stream that was current when the DeviceFile was made, a lazily allocated
    pinned bounce buffer, a lock, a byte counter."""

    device_type = "cuda"

    def __init__(self, tensors, bounce_bytes: int):
        import torch

        self._attach(tensors, bounce_bytes)
        device = self.segments[0].device
        self.stream = torch.cuda.Stream(device)
        # everything already queued on the caller's stream (the kernels that produced the tensors) runs first
        self.stream.wait_stream(torch.cuda.current_stream(device))
        self.stream_handle = self.stream.cuda_stream

    def _attach(self, tensors, bounce_bytes: int):
        """``tensors``: one tensor, or a non-empty list of them in file order."""
        import torch

        self.tensors = list(tensors) if isinstance(tensors, (list, tuple)) else [tensors]  # keep the storages alive
        self.segments = [t.reshape(-1).view(torch.uint8) for t in self.tensors]
        self.seg_start = [0]  # file offset of every segment, then the size
        for s in self.segments:
            self.seg_start.append(self.seg_start[-1] + s.numel())
        self.nbytes = self.seg_start[-1]
        self.lock = threading.Lock()
        self.bytes_to_host = 0
        self._bounce_bytes = max(1, min(bounce_bytes, self.nbytes))
        self._bounce = None

    # the device-specific steps (the CPU tests replace these)
    def _on_stream(self):
        import torch

        return torch.cuda.stream(self.stream)

    def _new_bounce(self, n: int):
        import torch

        return torch.empty(n, dtype=torch.uint8, pin_memory=True)

    def _wait(self):
        self.stream.synchronize()

    def _after(self, other: "_TensorBytes"):
        """Order this source's stream after everything ``other``'s stream holds."""
        if other.stream_handle != self.stream_handle:
            self.stream.wait_stream(other.stream)

    @classmethod
    def _to_device(cls, data: bytes, ctx):
        import torch

        return torch.frombuffer(bytearray(data), dtype=torch.uint8).to(f"cuda:{ctx.device}")

    @classmethod
    def _check_tensor(cls, tensor, ctx, label: str):
        """Raises ``ValueError`` unless ``tensor`` can be a segment; returns the context (``get_context()`` if None)."""
        if getattr(getattr(tensor, "device", None), "type", None) != cls.device_type:
            raise ValueError(f"{label} needs a CUDA tensor")
        if not tensor.is_contiguous():
            raise ValueError(f"{label} needs a contiguous tensor")
        ctx = ctx or get_context()
        if getattr(ctx, "device", tensor.device.index) not in (tensor.device.index, -1):
            raise ValueError(f"{label}: tensor lives on cuda:{tensor.device.index} but the context is bound to "
                             f"cuda:{ctx.device}")
        return ctx

    def copy_out(self, pos: int, dst: np.ndarray) -> None:
        """dst[:] = bytes [pos, pos + dst.size) of the file, one bounce buffer at a time (a bounce buffer may be filled
        from several segments)."""
        n = int(dst.size)
        with self.lock:
            if self._bounce is None:
                self._bounce = self._new_bounce(self._bounce_bytes)
            bounce = self._bounce.numpy()
            done = 0
            seg = bisect.bisect_right(self.seg_start, pos) - 1
            while done < n:
                k = min(n - done, self._bounce_bytes)
                filled = 0
                with self._on_stream():
                    while filled < k:
                        at = pos + done + filled
                        while self.seg_start[seg + 1] <= at:  # skips empty segments
                            seg += 1
                        lo = at - self.seg_start[seg]
                        m = min(k - filled, self.seg_start[seg + 1] - at)
                        self._bounce[filled : filled + m].copy_(self.segments[seg][lo : lo + m], non_blocking=True)
                        filled += m
                self._wait()
                dst[done : done + k] = bounce[:k]
                done += k
            self.bytes_to_host += n

    def hash_parts(self, ctx, part_len: int, flags: int):
        """``Context.hash_fixed_parts`` over the bytes where they are; only the digest table comes back."""
        if part_len <= 0:
            raise ValueError("part_len must be > 0")
        if len(self.segments) > 1:
            return _hash_sources([self], ctx, part_len, flags)
        n = -(-self.nbytes // part_len)
        with self.lock, self._on_stream():
            d_sha, d_md5, d_trim = _outputs(n, flags, self.segments[0].device)
            got = ctx.hash_fixed_parts_device(self.segments[0].data_ptr(), self.nbytes, part_len, flags, _ptr(d_sha),
                                              _ptr(d_md5), _ptr(d_trim), 0, self.stream_handle)
            assert got == n
            return _fetch(d_sha, d_md5, d_trim)


def _outputs(n: int, flags: int, device):
    import torch

    d_sha = torch.empty((n, 32), dtype=torch.uint8, device=device) if flags & _lib.SHA256 else None
    d_md5 = torch.empty((n, 16), dtype=torch.uint8, device=device) if flags & _lib.MD5 else None
    return d_sha, d_md5, torch.empty(n, dtype=torch.int64, device=device)


def _fetch(d_sha, d_md5, d_trim):
    # .cpu() on the current stream: the copies follow the hash launches and return once the table is on the host
    sha = d_sha.cpu().numpy() if d_sha is not None else None
    md5 = d_md5.cpu().numpy() if d_md5 is not None else None
    return sha, md5, d_trim.cpu().numpy().astype(np.uint64)


def _ptr(t) -> int:
    return t.data_ptr() if t is not None and t.numel() else 0


def _hash_sources(sources: list[_TensorBytes], ctx, part_len: int, flags: int):
    if part_len <= 0:
        raise ValueError("part_len must be > 0")
    lead = sources[0]
    ptrs, lens, first = [], [], [0]
    for src in sources:
        lead._after(src)
        ptrs += [s.data_ptr() if s.numel() else 0 for s in src.segments]
        lens += [s.numel() for s in src.segments]
        first.append(len(lens))
    n = sum(-(-src.nbytes // part_len) for src in sources)
    with lead._on_stream():
        d_sha, d_md5, d_trim = _outputs(n, flags, lead.segments[0].device)
        got = ctx.hash_segment_parts_device(ptrs, lens, first, part_len, flags, _ptr(d_sha), _ptr(d_md5), _ptr(d_trim),
                                            lead.stream_handle)
        assert got == n
        return _fetch(d_sha, d_md5, d_trim)


def hash_parts_many(files: list["DeviceFile"], part_len: int, flags: int = _lib.SHA256 | _lib.MD5, ctx=None):
    """``DeviceFile.hash_parts`` of several files at once: every file's parts (one or more segments each), file-major,
    digested by ONE ``b200h_hash_segment_parts_device`` call on the first file's stream, which is ordered after every
    file's stream.  -> (sha uint8[n,32] | None, md5 uint8[n,16] | None, trimmed uint64[n])."""
    return _hash_sources([f._src for f in files], ctx or get_context(), part_len, flags)


# ------------------------------------------------------------------------------------------ safetensors

# safetensors dtype tags by torch dtype name, in the order ``safetensors.torch.save`` lays tensor data out: the higher
# the rank the earlier, ties by name (tests/test_segment_parts_cpu.py pins this against the library)
_ST_TAGS = (
    ("bool", "BOOL"), ("float4_e2m1fn_x2", "F4"), ("uint8", "U8"), ("int8", "I8"), ("float8_e5m2", "F8_E5M2"),
    ("float8_e4m3fn", "F8_E4M3"), ("float8_e8m0fnu", "F8_E8M0"), ("int16", "I16"), ("uint16", "U16"),
    ("float16", "F16"), ("bfloat16", "BF16"), ("int32", "I32"), ("uint32", "U32"), ("float32", "F32"),
    ("complex64", "C64"), ("float64", "F64"), ("int64", "I64"), ("uint64", "U64"),
)


def _st_dtypes() -> dict:
    """torch dtype -> (tag, rank) for the dtypes this torch has."""
    import torch

    return {getattr(torch, name): (tag, rank) for rank, (name, tag) in enumerate(_ST_TAGS) if hasattr(torch, name)}


def safetensors_layout(tensors: Mapping, metadata: Mapping | None = None):
    """(header bytes, [(name, tensor), ...] in data order) of the safetensors image of ``tensors``: the 8-byte
    little-endian header length, the compact JSON header (``__metadata__`` first when given, then every tensor's
    dtype / shape / data_offsets in data order), padded with spaces to a multiple of 8.  Checks names, metadata and
    dtypes (``ValueError``); where the tensors live is the caller's business."""
    import torch

    if not isinstance(tensors, Mapping):
        raise ValueError(f"expected a mapping of str -> torch.Tensor, got {type(tensors).__name__}")
    if metadata is not None:
        if not isinstance(metadata, Mapping):
            raise ValueError(f"metadata must be a mapping of str -> str, got {type(metadata).__name__}")
        for k, v in metadata.items():
            if not isinstance(k, str) or not isinstance(v, str):
                raise ValueError(f"metadata entries must be str -> str, got {k!r}: {v!r}")
    dtypes = _st_dtypes()
    for name, t in tensors.items():
        if not isinstance(name, str):
            raise ValueError(f"tensor names must be str, got {name!r}")
        if name == "__metadata__":
            raise ValueError("'__metadata__' is reserved for the header's metadata and cannot name a tensor")
        if not isinstance(t, torch.Tensor) or t.layout != torch.strided:
            raise ValueError(f"{name!r} is not a dense torch.Tensor")
        if t.dtype not in dtypes:
            raise ValueError(f"{name!r} has dtype {t.dtype}, which safetensors cannot store")
        if dtypes[t.dtype][0] == "F4" and t.dim() == 0:
            raise ValueError(f"{name!r}: a 0-d {t.dtype} tensor has no safetensors shape")
    ordered = sorted(tensors.items(), key=lambda kv: (-dtypes[kv[1].dtype][1], kv[0]))
    header: dict = {}
    if metadata is not None:
        header["__metadata__"] = dict(metadata)
    at = 0
    for name, t in ordered:
        tag = dtypes[t.dtype][0]
        shape = list(t.shape)
        if tag == "F4":  # two 4-bit values per element: safetensors counts values
            shape[-1] *= 2
        n = t.numel() * t.element_size()
        header[name] = {"dtype": tag, "shape": shape, "data_offsets": [at, at + n]}
        at += n
    text = json.dumps(header, ensure_ascii=False, separators=(",", ":")).encode("utf-8")
    text += b" " * (-len(text) % 8)
    return len(text).to_bytes(8, "little") + text, ordered


class DeviceFile(io.RawIOBase):
    """Read-only, seekable ``BinaryIO`` over the raw bytes of one contiguous CUDA tensor (any dtype), in memory order,
    or (``DeviceFile.safetensors``) over the safetensors image of many.

    ``fileno()`` raises ``OSError`` (there is no descriptor).  Reads are ordered after the work that was queued on the
    current CUDA stream when the DeviceFile was made; the tensors are kept alive by it."""

    _Source = _TensorBytes

    def __init__(self, tensor, *, ctx=None, bounce_bytes: int = BOUNCE_BYTES):
        super().__init__()
        self._Source._check_tensor(tensor, ctx, "DeviceFile")
        self._src = self._Source(tensor, bounce_bytes)
        self._pos = 0

    @classmethod
    def safetensors(cls, tensors: Mapping, metadata: Mapping | None = None, *, ctx=None,
                    bounce_bytes: int = BOUNCE_BYTES) -> "DeviceFile":
        """A file whose bytes are the safetensors image of ``tensors`` (``safetensors.torch.save(tensors, metadata)``),
        made of the tensors where they are: the header is built on the host and copied to the device once, every tensor
        is one segment of the file.  Tensors must be contiguous, on the context's device, of a dtype safetensors stores;
        zero-size, 0-d and storage-sharing tensors are fine.  The metadata entries keep the mapping's order (the
        library writes them in no fixed order when there are several)."""
        header, ordered = safetensors_layout(tensors, metadata)
        for name, t in ordered:
            ctx = cls._Source._check_tensor(t, ctx, f"DeviceFile.safetensors[{name!r}]")
        head = cls._Source._to_device(header, ctx or get_context())
        return cls._over(cls._Source([head] + [t for _, t in ordered], bounce_bytes))

    @classmethod
    def _over(cls, src) -> "DeviceFile":
        f = cls.__new__(cls)
        io.RawIOBase.__init__(f)
        f._src, f._pos = src, 0
        return f

    @property
    def nbytes(self) -> int:
        """Size of the file in bytes."""
        return self._src.nbytes

    @property
    def bytes_to_host(self) -> int:
        """Bytes copied device -> host by this file and every reader ``reopen()`` made from it."""
        return self._src.bytes_to_host

    def reopen(self) -> "DeviceFile":
        """An independent reader (own position) over the same bytes, bounce buffer and ``bytes_to_host`` counter."""
        return DeviceFile._over(self._src)

    def hash_parts(self, part_len: int, flags: int = _lib.SHA256 | _lib.MD5, ctx=None):
        """Split the bytes into ceil(size / part_len) parts and digest them where they are
        (``b200h_hash_fixed_parts_device`` for one tensor, ``b200h_hash_segment_parts_device`` for several).
        -> (sha uint8[n,32] | None, md5 uint8[n,16] | None, trimmed uint64[n]); nothing but this table leaves the
        device."""
        return self._src.hash_parts(ctx or get_context(), part_len, flags)

    # ---- BinaryIO
    def readable(self) -> bool:
        return True

    def seekable(self) -> bool:
        return True

    def fileno(self) -> int:
        raise io.UnsupportedOperation("DeviceFile has no file descriptor (its bytes are in GPU memory)")

    def tell(self) -> int:
        self._check_open()
        return self._pos

    def seek(self, offset: int, whence: int = os.SEEK_SET) -> int:
        self._check_open()
        if whence == os.SEEK_SET:
            pos = offset
        elif whence == os.SEEK_CUR:
            pos = self._pos + offset
        elif whence == os.SEEK_END:
            pos = self._src.nbytes + offset
        else:
            raise ValueError(f"invalid whence ({whence})")
        if pos < 0:
            raise ValueError(f"negative seek position {pos}")
        self._pos = pos
        return pos

    def readinto(self, b) -> int:
        self._check_open()
        dst = np.frombuffer(memoryview(b).cast("B"), dtype=np.uint8)
        n = max(0, min(dst.size, self._src.nbytes - self._pos))
        if n:
            self._src.copy_out(self._pos, dst[:n])
            self._pos += n
        return n

    def read(self, size: int | None = -1) -> bytes:
        self._check_open()
        left = max(0, self._src.nbytes - self._pos)
        n = left if size is None or size < 0 else min(size, left)
        out = bytearray(n)
        if n:
            self._src.copy_out(self._pos, np.frombuffer(out, dtype=np.uint8))
            self._pos += n
        return bytes(out)

    def readall(self) -> bytes:
        return self.read(-1)

    def _check_open(self):
        if self.closed:
            raise ValueError("I/O operation on closed DeviceFile")

    def __repr__(self) -> str:
        segs = self._src.tensors
        if len(segs) == 1:
            return f"<DeviceFile {self._src.nbytes} bytes of {segs[0].dtype} on {segs[0].device}>"
        return f"<DeviceFile {self._src.nbytes} bytes in {len(segs)} segments on {segs[0].device}>"


__all__ = ["DeviceFile", "BOUNCE_BYTES", "hash_parts_many", "safetensors_layout"]
