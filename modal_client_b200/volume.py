"""``Volume.batch_upload()`` on the GPU hash path.

Counterparts of ``_VolumeUploadContextManager`` (volumefs1: whole-file SHA-256 + MD5, dedupe through
``MountPutFile``, py/modal/volume.py:1181-1333) and ``_VolumeUploadContextManager2`` (volumefs2: SHA-256 of every
zero-trimmed 8 MiB block, ``VolumePutFiles2`` missing-block loop, :1345-1574).  Same ``put_file`` /
``put_directory`` surface and the same RPC / PUT sequence; what changes is *when hashing happens*: the reference
hashes file by file (ThreadPoolExecutor) or block by block (``to_thread`` under a semaphore); here every path
queued in the batch is handed to ``blob_utils.get_file_upload_specs`` / ``file_upload_specs2`` -- ONE GPU
batch for the whole tree -- before the first RPC goes out.  File objects (``BytesIO`` / open files) keep the
per-object spec builders.  A ``DeviceFile`` (the bytes of a CUDA tensor) is hashed in GPU memory by the volumefs2
uploader -- all of a batch's ``DeviceFile``s, safetensors images of whole state dicts included, in one device call
(``blob_utils.device_file_specs2``) -- and only the trimmed bytes of the blocks the server is missing are copied to the
host; the volumefs1 uploader reads it like any other stream.  Given ``device_staging_bytes`` of page-locked host memory,
the volumefs2 uploader copies those blocks off the device in waves of one ``stage_ranges`` call each and PUTs them from
there, so the tensors are free again (``device_released``) after the last copy instead of after the last PUT.
"""
from __future__ import annotations

import asyncio
import functools
import os
import time
from collections.abc import Callable
from io import BytesIO
from pathlib import Path, PurePosixPath
from typing import Any, BinaryIO

import numpy as np

from . import _wire, blob_utils
from ._logging import logger
from .async_utils import bounded_map, retry
from .blob_utils import FileUploadSpec, FileUploadSpec2, _ByteBudget
from .device_file import DeviceFile, stage_ranges
from .exception import ExecutionError
from .http_utils import ClientSessionRegistry

VOLUME_PUT_FILE_CLIENT_TIMEOUT = 60 * 60  # seconds a single file may take to become visible (volume.py:79)


class VolumeUploadTimeoutError(TimeoutError):
    pass


class _BatchBase:
    def __init__(self, volume_id: str, client, progress_cb: Callable[..., Any] | None = None, force: bool = False):
        self._volume_id = volume_id
        self._client = client
        self._progress_cb = progress_cb or (lambda *_, **__: None)
        self._force = force
        self._paths: list[tuple[Path | str, str, int | None]] = []  # (local path, remote posix path, mode)
        self._fileobjs: list[tuple[BinaryIO, PurePosixPath, int]] = []

    async def __aenter__(self):
        return self

    def put_file(self, local_file: Path | str | BinaryIO | BytesIO, remote_path: PurePosixPath | str, mode: int | None = None):
        """Queue one file (path or readable file object, ``DeviceFile`` included; objects must stay readable and
        unchanged until the batch exits)."""
        remote = PurePosixPath(remote_path).as_posix()
        if remote.endswith("/"):
            raise ValueError(f"remote_path ({remote}) must refer to a file - cannot end with /")
        if isinstance(local_file, (str, Path)):
            self._paths.append((local_file, remote, mode))
        else:
            self._fileobjs.append((local_file, PurePosixPath(remote), mode or 0o644))

    def put_directory(self, local_path: Path | str, remote_path: PurePosixPath | str, recursive: bool = True):
        """Queue every regular file below ``local_path`` (directories and special files are skipped).

        Same selection as the reference's ``rglob("*")`` + ``is_file()`` (py/modal/volume.py:1279-1284): symlinks to
        files count, symlinked directories are not descended into, fifos / devices are skipped.  The walk itself is
        ``os.scandir`` on plain strings: with hashing down to a fraction of a second, ``pathlib``'s ~15 us per file
        (glob + ``is_file`` + ``relative_to`` + ``/``) would be most of a million-file upload."""
        local_path = Path(local_path)
        assert local_path.is_dir()
        remote_root = PurePosixPath(remote_path).as_posix().rstrip("/")
        append = self._paths.append
        for abs_path, rel_posix in _walk_files(os.fspath(local_path), recursive):
            append((abs_path, f"{remote_root}/{rel_posix}", None))


def _walk_files(root: str, recursive: bool):
    """Yield (absolute path, path relative to ``root`` in posix form) of every regular file (or symlink to one)."""
    stack = [(root, "")]
    sep_is_posix = os.sep == "/"
    while stack:
        d, rel = stack.pop()
        try:
            it = os.scandir(d)
        except OSError:
            continue  # vanished or unreadable directory: pathlib's glob skips those too
        with it:
            for e in it:
                name = e.name
                try:
                    if e.is_dir(follow_symlinks=False):
                        if recursive:
                            stack.append((e.path, f"{rel}{name}/"))
                    elif e.is_file():  # follows symlinks, like Path.is_file()
                        yield e.path, (f"{rel}{name}" if sep_is_posix else f"{rel}{name}".replace(os.sep, "/"))
                except OSError:
                    continue


class VolumeUploadContextManager(_BatchBase):
    """volumefs1 batch upload: one fused SHA-256+MD5 GPU batch over all queued paths, then dedupe + upload."""

    def __init__(self, volume_id: str, client, progress_cb=None, force: bool = False):
        super().__init__(volume_id, client, progress_cb, force)
        self._byte_budget = _ByteBudget.from_system_memory()

    async def __aexit__(self, exc_type, exc_val, exc_tb):
        if exc_val:
            return
        specs: list[FileUploadSpec] = await asyncio.to_thread(blob_utils.get_file_upload_specs, self._paths)
        for fp, remote, mode in self._fileobjs:
            specs.append(await asyncio.to_thread(blob_utils.get_file_upload_spec_from_fileobj, fp, remote, mode))
        logger.debug(f"Computed checksums for {len(specs)} files on the GPU")
        # In-batch dedupe on the digest table, computed on the GPU (b200h_dedupe_host; what Mount does with a set,
        # py/modal/mount.py:498,518-534): each distinct content is checked / uploaded once, however many paths carry
        # it; the other paths only appear in the file index.  20 uploads in flight, like the reference (volume.py:1220).
        first, _ = await asyncio.to_thread(blob_utils.first_occurrence_of_specs, specs)
        owners = [i for i, f in enumerate(first) if f == i]
        await bounded_map(owners, lambda i: self._upload_file(specs[i]), concurrency=20)
        for i, spec in enumerate(specs):
            if first[i] != i:  # a copy of something already sent: account for it in the progress display
                self._progress_cb(task_id=self._progress_cb(name=spec.mount_filename, size=spec.size), complete=True)
        files = [_wire.MountFile(filename=s.mount_filename, sha256_hex=s.sha256_hex, mode=s.mode) for s in specs]
        self._progress_cb(complete=True)
        request = _wire.VolumePutFilesRequest(volume_id=self._volume_id, files=files,
                                              disallow_overwrite_existing_files=not self._force)
        try:
            await self._client.stub.VolumePutFiles(request)
        except Exception as exc:
            if type(exc).__name__ == "AlreadyExistsError":
                raise FileExistsError(str(exc))
            raise

    async def _upload_file(self, spec: FileUploadSpec):
        task_id = self._progress_cb(name=spec.mount_filename, size=spec.size)
        stub = self._client.stub
        response = await stub.MountPutFile(_wire.MountPutFileRequest(sha256_hex=spec.sha256_hex))
        if response.exists:  # content-addressed dedupe: nothing to send
            self._progress_cb(task_id=task_id, complete=True)
        else:
            started = time.monotonic()
            if spec.use_blob:
                with spec.source() as fp:
                    blob_id = await blob_utils.blob_upload_file(
                        fp, stub, functools.partial(self._progress_cb, task_id), sha256_hex=spec.sha256_hex,
                        md5_hex=spec.md5_hex, byte_budget=self._byte_budget)
                request2 = _wire.MountPutFileRequest(data_blob_id=blob_id, sha256_hex=spec.sha256_hex)
            else:
                content = spec.content if spec.content is not None else await asyncio.to_thread(spec.read_content)
                request2 = _wire.MountPutFileRequest(data=content, sha256_hex=spec.sha256_hex)
                self._progress_cb(task_id=task_id, complete=True)
            while True:
                response = await stub.MountPutFile(request2)
                if response.exists:
                    break
                if time.monotonic() - started >= VOLUME_PUT_FILE_CLIENT_TIMEOUT:
                    raise VolumeUploadTimeoutError(f"Uploading of {spec.source_description} timed out")
        return _wire.MountFile(filename=spec.mount_filename, sha256_hex=spec.sha256_hex, mode=spec.mode)


class VolumeUploadContextManager2(_BatchBase):
    """volumefs2 batch upload: all 8 MiB blocks of all queued files form one GPU batch (trim scan + SHA-256)."""

    def __init__(self, volume_id: str, client, progress_cb=None, force: bool = False,
                 hash_concurrency: int | None = None, put_concurrency: int = 128,
                 device_staging_bytes: int | None = None):
        """``device_staging_bytes``: page-locked host memory the batch may take (``ctx.host_alloc``, from the first
        missing-block answer until the batch ends) to stage the missing blocks of its ``DeviceFile``s: they are copied
        off the device in waves of at most half that many bytes, one device call per wave, and PUT from host memory,
        wave k + 1 being copied while wave k's PUTs run.  ``device_released`` is set once the last wave's copy has
        completed: from then on the batch never reads the tensors again, so they may change while the PUTs drain.  It
        must hold two blocks.  ``None`` (the default) takes no such memory: every block is read through its file's
        bounce buffer while it is PUT, and the tensors must not change until the batch has ended."""
        super().__init__(volume_id, client, progress_cb, force)
        # the reference hashes blocks under a semaphore of ``hash_concurrency`` = cpu_count executor threads
        # (volume.py:1358,1383); here every block of every file is one GPU batch, so the knob is accepted and unused
        self._hash_concurrency = hash_concurrency
        self._put_concurrency = put_concurrency
        if device_staging_bytes is not None and device_staging_bytes < 2 * blob_utils.BLOCK_SIZE:
            raise ValueError(f"device_staging_bytes must hold two blocks ({2 * blob_utils.BLOCK_SIZE} bytes), "
                             f"got {device_staging_bytes}")
        self._device_staging_bytes = device_staging_bytes
        self._device_files: dict[int, DeviceFile] = {}  # index into the batch's specs -> the file behind it
        self.device_released = asyncio.Event()  # the batch no longer reads its DeviceFiles' tensors

    async def __aexit__(self, exc_type, exc_val, exc_tb):
        if exc_val:
            return
        specs: list[FileUploadSpec2] = await blob_utils.file_upload_specs2(self._paths)
        # every DeviceFile of the batch: one device call; the specs keep put_file order
        device_specs = iter(await blob_utils.device_file_specs2([o for o in self._fileobjs if isinstance(o[0], DeviceFile)]))
        one_at_a_time = asyncio.Semaphore(1)
        for fp, remote, mode in self._fileobjs:
            if isinstance(fp, DeviceFile):
                self._device_files[len(specs)] = fp
                specs.append(next(device_specs))
            else:
                specs.append(await FileUploadSpec2.from_fileobj(fp, remote, one_at_a_time, mode))
        await self._put_file_specs(specs)

    async def _put_file_specs(self, file_specs: list[FileUploadSpec2]):
        staging = None
        if self._device_staging_bytes is not None:
            staging = _DeviceStaging(self._device_files, self._device_staging_bytes, self.device_released)
        try:
            await self._put_rounds(file_specs, staging)
        finally:
            if staging is not None:
                staging.close()
            self.device_released.set()  # at the latest when the batch ends, however it ends

    async def _put_rounds(self, file_specs: list[FileUploadSpec2], staging: "_DeviceStaging | None"):
        put_responses: dict[bytes, bytes] = {}
        B = _wire.VolumePutFiles2Request
        for _attempt in range(2):  # once to learn the missing blocks, once more with every put_response
            files = [
                B.File(path=s.path, mode=s.mode, size=s.size,
                       blocks=[B.Block(contents_sha256=b.contents_sha256, put_response=put_responses.get(b.contents_sha256))
                               for b in s.blocks])
                for s in file_specs
            ]
            request = B(volume_id=self._volume_id, files=files, disallow_overwrite_existing_files=not self._force)
            try:
                response = await self._client.stub.VolumePutFiles2(request)
            except Exception as exc:
                if type(exc).__name__ == "AlreadyExistsError":
                    raise FileExistsError(str(exc))
                raise
            if staging is not None:
                if not any(mb.file_index in staging.files for mb in response.missing_blocks):
                    self.device_released.set()
                elif self.device_released.is_set():
                    # the tensors were given back after the first round: there is nothing left to read
                    raise RuntimeError("Did not succeed at uploading all files despite supplying all missing blocks")
            if not response.missing_blocks:
                break
            await _put_missing_blocks(file_specs, response.missing_blocks, put_responses, self._put_concurrency,
                                      self._progress_cb, staging)
        else:
            raise RuntimeError("Did not succeed at uploading all files despite supplying all missing blocks")
        self._progress_cb(complete=True)


class _DeviceStaging:
    """The page-locked buffer a volumefs2 batch stages its DeviceFiles' missing blocks through: two halves, a wave of
    blocks each (every block at a multiple of 128 bytes, its trimmed length)."""

    ALIGN = 128

    def __init__(self, files: dict[int, DeviceFile], nbytes: int, released: asyncio.Event):
        self.files, self.released = files, released
        self.half = nbytes // 2 // self.ALIGN * self.ALIGN
        self._ctx, self._buf = None, None

    def buffer(self) -> np.ndarray:
        if self._buf is None:
            self._ctx = blob_utils.get_context()
            self._buf = self._ctx.host_alloc(2 * self.half)
        return self._buf

    def waves(self, file_specs, missing) -> list[list[tuple[Any, int, int]]]:
        """``missing`` (blocks of device files) cut greedily, in order, into waves that fit one half:
        [(missing block, offset in the half, trimmed length), ...] per wave."""
        waves, used = [], 0
        for mb in missing:
            block = file_specs[mb.file_index].blocks[mb.block_index]
            n = block.end - block.start
            if not waves or used + n > self.half:
                waves.append([])
                used = 0
            waves[-1].append((mb, used, n))
            used += -(-n // self.ALIGN) * self.ALIGN
        return waves

    def stage(self, file_specs, wave, half: int):
        """Enqueue one wave's copy into half ``half``: one ``stage_ranges`` call."""
        order = sorted({mb.file_index for mb, _, _ in wave})
        slot = {f: i for i, f in enumerate(order)}
        ranges = [(slot[mb.file_index], file_specs[mb.file_index].blocks[mb.block_index].start, n) for mb, _, n in wave]
        return stage_ranges([self.files[f] for f in order], ranges, self.buffer(),
                            [half * self.half + at for _, at, _ in wave], ctx=self._ctx)

    def close(self):
        if self._buf is not None:
            self._ctx.host_free(self._buf)
            self._buf = None


async def _put_missing_blocks(file_specs, missing_blocks, put_responses: dict[bytes, bytes], put_concurrency: int,
                              progress_cb: Callable[..., Any], staging: _DeviceStaging | None = None):
    """PUT each block the server reported missing (only the zero-trimmed bytes travel) and remember the
    server's put_response per block digest (py/modal/volume.py:1500-1574).  With ``staging``, the blocks of its device
    files are first copied to its buffer, a wave per device call, and sent from there; everything else about the round
    is the same."""
    from .bytes_io_segment_payload import BytesIOSegmentPayload, MemorySegmentPayload

    pending: dict[str, tuple[Any, set[int]]] = {}

    async def put_one(mb, staged_bytes: memoryview | None = None) -> tuple[bytes, bytes]:
        spec = file_specs[mb.file_index]
        block = spec.blocks[mb.block_index]
        if spec.path not in pending:
            pending[spec.path] = (progress_cb(name=spec.path, size=spec.size), set())
        task_id, waiting = pending[spec.path]
        waiting.add(mb.block_index)
        report = functools.partial(progress_cb, task_id=task_id)

        @retry(n_attempts=11, base_delay=0.5, attempt_timeout=None)  # reference: volume.py:1542
        async def attempt(payload) -> bytes:
            with payload.reset_on_error(subtract_progress=True):
                async with ClientSessionRegistry.get_session().put(mb.put_url, data=payload) as resp:
                    if resp.status != 200:
                        raise ExecutionError(f"block PUT failed with status {resp.status}: {await resp.text()}")
                    return await resp.content.read()

        if staged_bytes is not None:  # the block is in host memory already: sent from there, retries included
            data = await attempt(MemorySegmentPayload(staged_bytes, chunk_size=256 * 1024, progress_report_cb=report))
        else:
            with spec.source() as fp:
                # the block digest is already known (GPU batch): no re-hash while sending
                payload = BytesIOSegmentPayload(fp, block.start, block.end - block.start, chunk_size=256 * 1024,
                                                progress_report_cb=report, md5_digest=b"\0" * 16)
                data = await attempt(payload)
        waiting.discard(mb.block_index)
        if not waiting:
            report(complete=True)
        return block.contents_sha256, data

    # Identical blocks (the same content in several files, repeated runs inside one file) are sent once per round: the
    # put_response is kept per digest anyway (py/modal/volume.py:1464,1569).  First occurrences come from the GPU
    # dedupe over the digests of the missing blocks; the reference uploads every listed block.
    missing = list(missing_blocks)
    if len(missing) > 1:
        keys = np.frombuffer(b"".join(file_specs[mb.file_index].blocks[mb.block_index].contents_sha256 for mb in missing),
                             np.uint8).reshape(len(missing), 32)
        first, _ = await asyncio.to_thread(blob_utils.get_context().dedupe, keys)
        missing = [mb for i, mb in enumerate(missing) if first[i] == i]
    if staging is None:
        for digest, resp in await bounded_map(missing, put_one, concurrency=put_concurrency):
            put_responses[digest] = resp
        return

    slots = asyncio.Semaphore(put_concurrency)  # one bound for the staged and the unstaged PUTs of the round

    async def put_limited(item) -> tuple[bytes, bytes]:
        async with slots:
            return await put_one(*item)

    def start(items):
        return asyncio.ensure_future(bounded_map(items, put_limited, concurrency=put_concurrency))

    waves = staging.waves(file_specs, [mb for mb in missing if mb.file_index in staging.files])
    running = [start([(mb,) for mb in missing if mb.file_index not in staging.files])]
    if not waves:  # every missing device block has the content of an ordinary file's block that is sent instead
        staging.released.set()
    in_half: list[Any] = [None, None]  # the PUTs that still send from each half
    try:
        for k, wave in enumerate(waves):
            if in_half[k & 1] is not None:
                await in_half[k & 1]  # the half is free once every PUT out of it has its put_response
            staged = staging.stage(file_specs, wave, k & 1)
            await asyncio.to_thread(staged.wait)
            if k == len(waves) - 1:
                staging.released.set()
            in_half[k & 1] = start([(mb, staged.view(i)) for i, (mb, _, _) in enumerate(wave)])
            running.append(in_half[k & 1])
        for task in running:
            for digest, resp in await task:
                put_responses[digest] = resp
    finally:
        for task in running:
            task.cancel()
        await asyncio.gather(*running, return_exceptions=True)


# ---------------------------------------------------------------------------------- the reference's names

# enum VolumeFsVersion, modal_proto/api.proto:312-316
VOLUME_FS_VERSION_UNSPECIFIED, VOLUME_FS_VERSION_V1, VOLUME_FS_VERSION_V2 = 0, 1, 2


class _AbstractVolumeUploadContextManager:
    """The interface ``Volume.batch_upload`` hands out, and the version switch behind it (py/modal/volume.py:1137-1173)."""

    async def __aenter__(self): ...

    async def __aexit__(self, exc_type, exc_val, exc_tb): ...

    def put_file(self, local_file, remote_path, mode=None): ...

    def put_directory(self, local_path, remote_path, recursive=True): ...

    @staticmethod
    def resolve(version, object_id: str, client, progress_cb: Callable[..., Any] | None = None, force: bool = False,
                device_staging_bytes: int | None = None):
        """``device_staging_bytes`` goes to the volumefs2 manager only: volumefs1 needs whole-object digests and reads
        device files through the host anyway."""
        if version in (None, VOLUME_FS_VERSION_UNSPECIFIED, VOLUME_FS_VERSION_V1):
            return VolumeUploadContextManager(object_id, client, progress_cb=progress_cb, force=force)
        if version == VOLUME_FS_VERSION_V2:
            return VolumeUploadContextManager2(object_id, client, progress_cb=progress_cb, force=force,
                                               device_staging_bytes=device_staging_bytes)
        raise RuntimeError(f"unsupported volume version: {version}")


# The reference keeps the implementation under the underscore name and exports a synchronicity wrapper under the plain
# one; there is no wrapper layer here, so both names mean the class itself.
AbstractVolumeUploadContextManager = _AbstractVolumeUploadContextManager
_VolumeUploadContextManager = VolumeUploadContextManager
_VolumeUploadContextManager2 = VolumeUploadContextManager2

