"""NetworkFileSystem uploads on the GPU hash path.

Counterpart of the data path of ``_NetworkFileSystem`` (py/modal/network_file_system.py): ``write_file`` (:217-260),
``read_file`` (:262-276), ``add_local_file`` (:291-305) and ``add_local_dir`` (:307-335).  The reference hashes every
file with ``get_sha256_hex`` on the event loop (:227) -- and again inside ``blob_upload_file`` for the MD5 of files
above ``LARGE_FILE_LIMIT`` -- one file at a time under ``async_map(..., concurrency=20)``.  Here ``add_local_dir``
selects the files with one ``os.scandir`` walk and hashes the whole directory in ONE GPU batch
(``blob_utils.get_file_upload_specs``: SHA-256 + MD5 in a single pass over the bytes); the RPC sequence per file is
the reference's (``SharedVolumePutFile`` polled until ``exists``, blob upload above the limit).

Out of scope (control plane): object creation / lookup / deletion, ``iterdir`` / ``listdir`` / ``remove_file``.
"""
from __future__ import annotations

import asyncio
import functools
import os
import time
from collections.abc import AsyncIterator, Callable
from pathlib import Path, PurePosixPath
from typing import Any, BinaryIO

from . import _wire, blob_utils
from .async_utils import bounded_map
from .blob_utils import LARGE_FILE_LIMIT, blob_iter, blob_upload_file
from .hash_utils import get_sha256_hex
from .volume import _walk_files

NETWORK_FILE_SYSTEM_PUT_FILE_CLIENT_TIMEOUT = 10 * 60  # seconds, without the upload to blob storage (:31-33)


class NetworkFileSystemUploader:
    """The upload / read methods of ``_NetworkFileSystem`` for the object ``object_id``, driven through ``client.stub``."""

    def __init__(self, object_id: str, client):
        self.object_id = object_id
        self._client = client

    async def _put_and_wait(self, req, remote_path: str) -> None:
        t0 = time.monotonic()
        while time.monotonic() - t0 < NETWORK_FILE_SYSTEM_PUT_FILE_CLIENT_TIMEOUT:
            response = await self._client.stub.SharedVolumePutFile(req)
            if response.exists:
                return
        raise TimeoutError(f"Uploading of {remote_path} timed out")

    async def write_file(self, remote_path: str, fp: BinaryIO, progress_cb: Callable[..., Any] | None = None) -> int:
        """Write from a file object to ``remote_path``, atomically (reference :217-260)."""
        progress_cb = progress_cb or (lambda *_, **__: None)
        sha_hash = get_sha256_hex(fp)  # GPU; the stream position is restored
        fp.seek(0, os.SEEK_END)
        data_size = fp.tell()
        fp.seek(0)
        return await self._write(remote_path, fp, data_size, sha_hash, None, progress_cb)

    async def _write(self, remote_path: str, fp: BinaryIO, data_size: int, sha_hash: str, md5_hex: str | None,
                     progress_cb: Callable[..., Any]) -> int:
        if data_size > LARGE_FILE_LIMIT:  # module global, looked up at call time (tests patch it, like the reference's)
            task_id = progress_cb(name=remote_path, size=data_size)
            blob_id = await blob_upload_file(fp, self._client.stub, functools.partial(progress_cb, task_id),
                                             sha256_hex=sha_hash, md5_hex=md5_hex)
            req = _wire.SharedVolumePutFileRequest(shared_volume_id=self.object_id, path=remote_path,
                                                   data_blob_id=blob_id, sha256_hex=sha_hash, resumable=True)
        else:
            req = _wire.SharedVolumePutFileRequest(shared_volume_id=self.object_id, path=remote_path, data=fp.read(),
                                                   resumable=True)
        await self._put_and_wait(req, remote_path)
        return data_size  # "might be better if this is returned from the server" (:260)

    async def read_file(self, path: str) -> AsyncIterator[bytes]:
        """Read a file back (reference :262-276): inline data or the blob, chunk by chunk."""
        req = _wire.SharedVolumeGetFileRequest(shared_volume_id=self.object_id, path=path)
        try:
            response = await self._client.stub.SharedVolumeGetFile(req)
        except Exception as exc:
            if type(exc).__name__ == "NotFoundError":
                raise FileNotFoundError(exc.args[0] if exc.args else path)
            raise
        if response.WhichOneof("data_oneof") == "data":
            yield response.data
        else:
            async for data in blob_iter(response.data_blob_id, self._client.stub):
                yield data

    async def add_local_file(self, local_path: Path | str, remote_path: str | PurePosixPath | None = None,
                             progress_cb: Callable[..., Any] | None = None) -> int:
        local_path = Path(local_path)
        remote = (PurePosixPath("/", local_path.name) if remote_path is None else PurePosixPath(remote_path)).as_posix()
        with local_path.open("rb") as local_file:
            return await self.write_file(remote, local_file, progress_cb=progress_cb)

    async def add_local_dir(self, local_path: Path | str, remote_path: str | PurePosixPath | None = None,
                            progress_cb: Callable[..., Any] | None = None, concurrency: int = 20) -> int:
        """Upload every regular file below ``local_path`` (reference :307-335, which walks with ``rglob`` and hashes
        per file).  One GPU batch yields the SHA-256 of every file and the MD5 the blob path needs; uploads then run
        ``concurrency`` at a time like the reference's ``async_map``.  Returns the number of bytes written."""
        _local_path = Path(local_path)
        remote_root = (PurePosixPath("/", _local_path.name) if remote_path is None else PurePosixPath(remote_path)).as_posix()
        assert _local_path.is_dir()
        progress = progress_cb or (lambda *_, **__: None)
        files = [(abs_path, f"{remote_root.rstrip('/')}/{rel}", None)
                 for abs_path, rel in _walk_files(os.fspath(_local_path), recursive=True)]
        specs = await asyncio.to_thread(blob_utils.get_file_upload_specs, files, False)

        async def one(spec) -> int:
            with spec.source() as fp:
                md5_hex = spec.md5_hex if blob_utils._is_real_md5_hex(spec.md5_hex) else None
                return await self._write(spec.mount_filename, fp, spec.size, spec.sha256_hex, md5_hex, progress)

        return sum(await bounded_map(specs, one, concurrency=concurrency))


__all__ = ["NETWORK_FILE_SYSTEM_PUT_FILE_CLIENT_TIMEOUT", "LARGE_FILE_LIMIT", "NetworkFileSystemUploader"]
