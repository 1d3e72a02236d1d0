"""A read-only file object over the bytes of one CUDA tensor.

``DeviceFile(t)`` lets a buffer that lives in GPU memory -- a checkpoint shard, a safetensors image, an embedding
table -- go wherever the upload functions accept a ``BinaryIO``, without first copying the whole buffer to host memory:

* volumefs2 (``VolumeUploadContextManager2.put_file`` / ``FileUploadSpec2.from_fileobj``) recognises it and trims and
  hashes its 8 MiB blocks in place with one ``b200h_hash_fixed_parts_device`` call (``hash_parts``); only the
  (trimmed length, SHA-256) table comes to the host, and afterwards only the trimmed bytes of the blocks the server
  reports missing are read.
* every other consumer (volumefs1 ``put_file``, ``get_file_upload_spec_from_fileobj``, ``blob_upload_file``) reads it
  like any other stream.  Those digests are one serial chain over the whole object and gain nothing from the GPU.

``read`` / ``readinto`` copy device -> host through one page-locked bounce buffer of bounded size (16 MiB by default),
so host memory never has to hold the tensor.  ``bytes_to_host`` counts what has crossed.  The readers ``reopen()`` hands
out share the tensor, the bounce buffer and that counter.  The tensor must not change while an upload reads it.
"""
from __future__ import annotations

import io
import os
import threading

import numpy as np

from . import _lib
from ._backend import get_context

BOUNCE_BYTES = 16 << 20  # page-locked host memory per DeviceFile (shared by its reopen() readers)


class _TensorBytes:
    """The bytes of one contiguous CUDA tensor, plus what reading them needs: a side stream ordered after the stream
    that was current when the DeviceFile was made, a lazily allocated pinned bounce buffer, a lock, a byte counter."""

    def __init__(self, tensor, bounce_bytes: int):
        import torch

        self._attach(tensor, bounce_bytes)
        self.stream = torch.cuda.Stream(tensor.device)
        # everything already queued on the caller's stream (the kernels that produced the tensor) runs first
        self.stream.wait_stream(torch.cuda.current_stream(tensor.device))
        self.stream_handle = self.stream.cuda_stream

    def _attach(self, tensor, bounce_bytes: int):
        import torch

        self.tensor = tensor  # keeps the storage alive as long as any reader exists
        self.nbytes = tensor.numel() * tensor.element_size()
        self.data_ptr = tensor.data_ptr()
        self.flat = tensor.reshape(-1).view(torch.uint8)
        self.lock = threading.Lock()
        self.bytes_to_host = 0
        self._bounce_bytes = max(1, min(bounce_bytes, self.nbytes))
        self._bounce = None

    # the device-specific steps (the CPU tests replace these three)
    def _on_stream(self):
        import torch

        return torch.cuda.stream(self.stream)

    def _new_bounce(self, n: int):
        import torch

        return torch.empty(n, dtype=torch.uint8, pin_memory=True)

    def _wait(self):
        self.stream.synchronize()

    def copy_out(self, pos: int, dst: np.ndarray) -> None:
        """dst[:] = bytes [pos, pos + dst.size) of the tensor, one bounce buffer at a time."""
        n = int(dst.size)
        with self.lock:
            if self._bounce is None:
                self._bounce = self._new_bounce(self._bounce_bytes)
            bounce = self._bounce.numpy()
            done = 0
            while done < n:
                k = min(n - done, self._bounce_bytes)
                with self._on_stream():
                    self._bounce[:k].copy_(self.flat[pos + done : pos + done + k], non_blocking=True)
                self._wait()
                dst[done : done + k] = bounce[:k]
                done += k
            self.bytes_to_host += n

    def hash_parts(self, ctx, part_len: int, flags: int):
        """``Context.hash_fixed_parts`` over the tensor where it is; only the digest table comes back."""
        import torch

        if part_len <= 0:
            raise ValueError("part_len must be > 0")
        n = -(-self.nbytes // part_len)
        dev = self.flat.device
        with self.lock, self._on_stream():
            d_sha = torch.empty((n, 32), dtype=torch.uint8, device=dev) if flags & _lib.SHA256 else None
            d_md5 = torch.empty((n, 16), dtype=torch.uint8, device=dev) if flags & _lib.MD5 else None
            d_trim = torch.empty(n, dtype=torch.int64, device=dev)
            got = ctx.hash_fixed_parts_device(self.data_ptr, self.nbytes, part_len, flags, _ptr(d_sha), _ptr(d_md5),
                                              _ptr(d_trim), 0, self.stream_handle)
            assert got == n
            # .cpu() on this stream: the copies follow the hash launches and return once the table is on the host
            sha = d_sha.cpu().numpy() if d_sha is not None else None
            md5 = d_md5.cpu().numpy() if d_md5 is not None else None
            trimmed = d_trim.cpu().numpy().astype(np.uint64)
        return sha, md5, trimmed


def _ptr(t) -> int:
    return t.data_ptr() if t is not None and t.numel() else 0


class DeviceFile(io.RawIOBase):
    """Read-only, seekable ``BinaryIO`` over the raw bytes of one contiguous CUDA tensor (any dtype), in memory order.

    ``fileno()`` raises ``OSError`` (there is no descriptor).  Reads are ordered after the work that was queued on the
    current CUDA stream when the DeviceFile was made; the tensor is kept alive by it."""

    def __init__(self, tensor, *, ctx=None, bounce_bytes: int = BOUNCE_BYTES):
        super().__init__()
        if not getattr(tensor, "is_cuda", False):
            raise ValueError("DeviceFile needs a CUDA tensor")
        if not tensor.is_contiguous():
            raise ValueError("DeviceFile needs a contiguous tensor")
        ctx = ctx or get_context()
        if getattr(ctx, "device", tensor.device.index) not in (tensor.device.index, -1):
            raise ValueError(f"tensor lives on cuda:{tensor.device.index} but the context is bound to cuda:{ctx.device}")
        self._src = _TensorBytes(tensor, bounce_bytes)
        self._pos = 0

    @classmethod
    def _over(cls, src) -> "DeviceFile":
        f = cls.__new__(cls)
        io.RawIOBase.__init__(f)
        f._src, f._pos = src, 0
        return f

    @property
    def bytes_to_host(self) -> int:
        """Bytes copied device -> host by this file and every reader ``reopen()`` made from it."""
        return self._src.bytes_to_host

    def reopen(self) -> "DeviceFile":
        """An independent reader (own position) over the same bytes, bounce buffer and ``bytes_to_host`` counter."""
        return DeviceFile._over(self._src)

    def hash_parts(self, part_len: int, flags: int = _lib.SHA256 | _lib.MD5, ctx=None):
        """Split the bytes into ceil(size / part_len) parts and digest them where they are
        (``b200h_hash_fixed_parts_device``).  -> (sha uint8[n,32] | None, md5 uint8[n,16] | None, trimmed uint64[n]);
        nothing but this table leaves the device."""
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
        t = self._src.tensor
        return f"<DeviceFile {self._src.nbytes} bytes of {t.dtype} on {t.device}>"


__all__ = ["DeviceFile", "BOUNCE_BYTES"]
