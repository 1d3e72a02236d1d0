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

The way back (counterparts of ``Volume.read_file`` / ``read_file_into_fileobj``, py/modal/volume.py:878-1000):
``read_file`` and ``read_file_into_fileobj`` through host memory, ``read_file_into_device`` straight into the tensors
of a ``DeviceFile`` (blocks downloaded into page-locked memory, a wave per ``load_ranges`` call), and
``read_safetensors``, a safetensors checkpoint back into CUDA tensors without a host copy of the file,
``read_safetensors_slices``, slices of its tensors (a tensor-parallel rank's rows or columns) downloading only the blocks
they touch, ``read_torch_save``, a torch.save checkpoint back into CUDA storages, its zip CRC-32s checked on the device,
and ``read_safetensors_sharded``, a checkpoint in the Hugging Face Hub's sharded layout (``model.safetensors.index.json``)
through one wave loop over the blocks of all its shards.
"""
from __future__ import annotations

import asyncio
import functools
import json
import os
import time
from collections.abc import Callable, Mapping
from io import BytesIO
from pathlib import Path, PurePosixPath
from typing import Any, BinaryIO

import numpy as np

from . import _wire, blob_utils, device_file
from ._logging import logger
from .async_utils import bounded_map, bounded_map_ordered, gather_cancel_on_error, retry
from .blob_utils import FileUploadSpec, FileUploadSpec2, _ByteBudget
from .device_file import (BOUNCE_BYTES, DeviceFile, _st_dtypes, cast_dtypes, cast_targets, fp8_dtypes, load_boxes,
                          load_cast_boxes, load_fp8_amax_boxes, load_quant_boxes, load_ranges, load_scaled_boxes,
                          stage_ranges)
from .exception import ExecutionError, ServiceError
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


# -------------------------------------------------------------------------------------------------- reads
#
# The read direction of volumefs2: ``VolumeGetFile2`` names the blocks that hold a byte range of a file, one GET URL
# per block, the first one sliced from ``start % BLOCK_SIZE`` and the last one cut at the end of the range; the server
# zero-pads a block that was stored trimmed, so every body has exactly its slice's length.


async def _raise_on_block_response_error(response) -> None:
    """An HTTP status >= 400 of a block GET as the reference reports it (py/modal/volume.py:82-99): 503 is a
    ``ServiceError``, anything else an ``ExecutionError``."""
    if response.status < 400:
        return
    try:
        body = await response.text()
    except Exception:
        body = "<unavailable>"
    if response.status == 503:
        raise ServiceError(f"Service temporarily unavailable: {body}")
    raise ExecutionError(f"Request failed with status {response.status} {response.reason}: {body}")


async def _get_file2(client, volume_id: str, path: str, start: int = 0, length: int = 0):
    try:
        return await client.stub.VolumeGetFile2(_wire.VolumeGetFile2Request(volume_id=volume_id, path=path, start=start,
                                                                             len=length))
    except Exception as exc:
        if type(exc).__name__ == "NotFoundError":
            raise FileNotFoundError(exc.args[0] if exc.args else path)
        raise


async def read_file(client, volume_id: str, path: str):
    """Async generator of the file's block bodies, in order (py/modal/volume.py:878-920): ``cpu_count`` blocks are
    fetched ahead, each GET is retried (5 attempts, 0.1 s base delay).  A missing path raises ``FileNotFoundError``."""
    response = await _get_file2(client, volume_id, path)

    @retry(n_attempts=5, base_delay=0.1, attempt_timeout=None)
    async def read_block(url: str) -> bytes:
        async with ClientSessionRegistry.get_session().get(url) as get_response:
            await _raise_on_block_response_error(get_response)
            return await get_response.content.read()

    async for body in bounded_map_ordered(list(response.get_urls), read_block, concurrency=os.cpu_count() or 1):
        yield body


async def read_file_into_fileobj(client, volume_id: str, path: str, fileobj: BinaryIO,
                                 progress_cb: Callable[..., Any] | None = None, concurrency: int | None = None) -> int:
    """Write the whole file into ``fileobj`` from its current position, ``concurrency`` (``cpu_count``) blocks at a
    time, each at its place in the file (py/modal/volume.py:923-1000); -> the number of bytes written.  Leaves the
    position behind the last byte.  ``progress_cb(advance=n)`` is called as bytes are written."""
    progress_cb = progress_cb or (lambda *_, **__: None)
    response = await _get_file2(client, volume_id, path)
    semaphore = asyncio.Semaphore(concurrency or os.cpu_count() or 1)
    write_lock = asyncio.Lock()
    start_pos = fileobj.tell()

    @retry(n_attempts=5, base_delay=0.1, attempt_timeout=None)
    async def download_block(idx: int, url: str) -> int:
        block_start_pos = start_pos + idx * blob_utils.BLOCK_SIZE
        written = 0
        async with semaphore, ClientSessionRegistry.get_session().get(url) as get_response:
            await _raise_on_block_response_error(get_response)
            async for chunk in get_response.content.iter_any():
                async with write_lock:
                    fileobj.seek(block_start_pos + written)
                    fileobj.write(chunk)
                progress_cb(advance=len(chunk))
                written += len(chunk)
        return written

    total = sum(await asyncio.gather(*[download_block(i, url) for i, url in enumerate(response.get_urls)]))
    fileobj.seek(start_pos + total)
    return total


async def _block_slices(client, volume_id: str, path: str, start: int, n: int) -> list[tuple[str, int, int]]:
    """[(GET URL, offset in the range, length), ...] of bytes [start, start + n) of the file, n > 0: one
    ``VolumeGetFile2`` call, whose answer is checked against the file's size and the block geometry before any GET."""
    BS = blob_utils.BLOCK_SIZE
    response = await _get_file2(client, volume_id, path, start, n)
    if start + n > response.size:
        raise ValueError(f"{path}: bytes [{start}, {start + n}) lie beyond the end of the file ({response.size} bytes)")
    if response.len != n:
        raise ExecutionError(f"{path}: asked for {n} bytes at {start}, the server answered with {response.len}")
    first, last = start // BS, (start + n - 1) // BS
    urls = list(response.get_urls)
    if len(urls) != last - first + 1:
        raise ExecutionError(f"{path}: bytes [{start}, {start + n}) span {last - first + 1} blocks, the server named "
                             f"{len(urls)}")
    out = []
    for k, url in enumerate(urls):
        lo, hi = max(start, (first + k) * BS), min(start + n, (first + k + 1) * BS)
        out.append((url, lo - start, hi - lo))
    return out


@retry(n_attempts=5, base_delay=0.1, attempt_timeout=None)
async def _fetch_block(url: str, out: np.ndarray, want: int, semaphore: asyncio.Semaphore) -> None:
    """out[:want] = the body of one block GET, which must be exactly ``want`` bytes long.  A retry starts over in the
    same place."""
    got = 0
    async with semaphore, ClientSessionRegistry.get_session().get(url) as response:
        await _raise_on_block_response_error(response)
        async for chunk in response.content.iter_any():
            if got + len(chunk) > want:
                raise ExecutionError(f"block GET returned more than the {want} bytes of its slice")
            out[got : got + len(chunk)] = np.frombuffer(chunk, np.uint8)
            got += len(chunk)
    if got != want:
        raise ExecutionError(f"block GET returned {got} bytes, its slice has {want}")


async def _read_range_host(client, volume_id: str, path: str, start: int, n: int) -> bytes:
    """Bytes [start, start + n) of the file, through host memory (small reads: a safetensors header)."""
    if n == 0:
        return b""
    out = np.empty(n, np.uint8)
    semaphore = asyncio.Semaphore(os.cpu_count() or 1)
    await gather_cancel_on_error(*[_fetch_block(url, out[at : at + m], m, semaphore)
                                   for url, at, m in await _block_slices(client, volume_id, path, start, n)])
    return out.tobytes()


async def read_file_into_device(client, volume_id: str, path: str, dst: DeviceFile, *, start: int = 0,
                                staging_bytes: int = 256 << 20, concurrency: int | None = None,
                                progress_cb: Callable[..., Any] | None = None) -> int:
    """Fill ``dst`` (a ``DeviceFile``: its tensors are written in place) with bytes [start, start + dst.nbytes) of the
    file; -> the number of bytes written.

    One ``VolumeGetFile2`` call names the blocks; its answer must match the size of ``dst`` and the block geometry, else
    this raises before any GET.  The blocks are fetched, ``concurrency`` (``cpu_count``) at a time, straight into slots
    of ``staging_bytes`` of page-locked memory (``ctx.host_alloc``, freed however the call ends) taken in two halves:
    when a half's wave of blocks is complete it goes to the device with one ``load_ranges`` call while the next wave
    downloads into the other half, and a half is refilled only after its previous copy has read it.  Each block body
    must have exactly its slice's length (the server zero-pads blocks that were stored trimmed), else
    ``ExecutionError`` after the GET's retries.  ``staging_bytes`` must hold two blocks (``ValueError``).
    On return the bytes are ordered before work enqueued later on the current stream.  If the call raises, ``dst``
    holds partial content: some of its bytes are the file's, the others what they were."""
    BS = blob_utils.BLOCK_SIZE
    if staging_bytes < 2 * BS:
        raise ValueError(f"staging_bytes must hold two blocks ({2 * BS} bytes), got {staging_bytes}")
    progress_cb = progress_cb or (lambda *_, **__: None)
    n = dst.nbytes
    if n == 0:
        await _get_file2(client, volume_id, path, start, 1)  # the file must exist; nothing else to do
        return 0
    slices = await _block_slices(client, volume_id, path, start, n)
    await _load_in_waves(slices, lambda wave, at, buf, ctx: load_ranges([dst], [(0, off, m) for _, off, m in wave], buf,
                                                                        at, ctx=ctx),
                         staging_bytes, concurrency, progress_cb)
    return n


async def _load_in_waves(slices, load, staging_bytes: int, concurrency: int | None,
                         progress_cb: Callable[..., Any]) -> None:
    """Download ``slices`` (``_block_slices``, each possibly followed by more fields that ``load`` reads) to the device:
    every block goes to its own ``BLOCK_SIZE`` slot of a page-locked buffer (``ctx.host_alloc``) of two halves, a wave
    per half; when a wave is complete,
    ``load(wave, at, buf, ctx)`` -- the wave's slices, their offsets in the buffer, the buffer and the context -- makes
    its one copy (``load_ranges`` or ``load_boxes``) and returns the ``Loaded``, or ``(Loaded, True)`` when its copies
    also read the previous wave's slots (a quantized band carried over from there).  A half is refilled only after
    every copy that reads it has read it, so ``load`` may still read the previous wave's slots; every copy has read the
    buffer before it is freed, however the call ends."""
    BS = blob_utils.BLOCK_SIZE
    per_half = staging_bytes // 2 // BS  # block slots per half (every slot starts at a multiple of BLOCK_SIZE)
    semaphore = asyncio.Semaphore(concurrency or os.cpu_count() or 1)
    ctx = blob_utils.get_context()
    buf = ctx.host_alloc(2 * per_half * BS)
    loaded: list = [None, None]
    try:
        for k, w in enumerate(range(0, len(slices), per_half)):
            wave, half = slices[w : w + per_half], k & 1
            if loaded[half] is not None:
                await asyncio.to_thread(loaded[half].wait)  # the half's previous copy has read it
                loaded[half] = None
            at = [(half * per_half + i) * BS for i in range(len(wave))]

            async def fetch(url: str, m: int, a: int):
                await _fetch_block(url, buf[a : a + m], m, semaphore)
                progress_cb(advance=m)

            await gather_cancel_on_error(*[fetch(url, m, a) for (url, _, m, *_), a in zip(wave, at)])
            got = load(wave, at, buf, ctx)
            loaded[half], carried = got if isinstance(got, tuple) else (got, False)
            if carried:  # the copy also read the previous wave's slots: that half is refilled only after it too
                loaded[1 - half] = loaded[half]
    finally:
        for pending in loaded:  # the copies must have read the buffer before it is freed
            if pending is not None:
                await asyncio.to_thread(pending.wait)
        ctx.host_free(buf)


def _safetensors_entries(header: bytes, data_len: int):
    """(``__metadata__`` or None, [(name, torch dtype, torch shape, start, end), ...] in data order), checked as the
    safetensors library checks a header (a valid JSON object, known dtype tags, ``shape x element size`` = span, ``data_offsets`` tiling the data
    region of ``data_len`` bytes without holes or overlap); ``ValueError`` otherwise."""
    try:
        meta = json.loads(header.decode("utf-8"))
    except (UnicodeDecodeError, ValueError) as exc:
        raise ValueError(f"safetensors header is not valid JSON: {exc}") from None
    if not isinstance(meta, dict):
        raise ValueError("safetensors header is not a JSON object")
    extra = meta.pop("__metadata__", None)
    if extra is not None and not (isinstance(extra, dict) and all(isinstance(v, str) for v in extra.values())):
        raise ValueError("safetensors __metadata__ must map str to str")
    by_tag = {tag: dtype for dtype, (tag, _) in _st_dtypes().items()}
    entries = []
    for name, info in meta.items():
        if not isinstance(info, dict) or set(info) != {"dtype", "shape", "data_offsets"}:
            raise ValueError(f"safetensors header: {name!r} needs exactly dtype, shape and data_offsets")
        tag, shape, offs = info["dtype"], info["shape"], info["data_offsets"]
        if tag not in by_tag:
            raise ValueError(f"safetensors header: {name!r} has dtype {tag!r}, which this torch cannot hold")
        ints = lambda v: isinstance(v, list) and all(isinstance(x, int) and not isinstance(x, bool) and x >= 0 for x in v)  # noqa: E731
        if not ints(shape) or not ints(offs) or len(offs) != 2:
            raise ValueError(f"safetensors header: {name!r} has a malformed shape or data_offsets")
        dtype, shape = by_tag[tag], list(shape)
        if tag == "F4":  # the header counts 4-bit values, the torch dtype holds two per element
            if not shape or shape[-1] % 2:
                raise ValueError(f"safetensors header: {name!r} is F4 with an odd or missing last dimension")
            shape[-1] //= 2
        size = dtype.itemsize
        for d in shape:
            size *= d
        if offs[1] < offs[0] or offs[1] - offs[0] != size:
            raise ValueError(f"safetensors header: {name!r} spans {offs[1] - offs[0]} bytes, its shape and dtype "
                             f"need {size}")
        entries.append((name, dtype, shape, offs[0], offs[1]))
    entries.sort(key=lambda e: (e[3], e[4]))
    at = 0
    for name, _, _, lo, hi in entries:
        if lo != at:
            raise ValueError(f"safetensors header: {name!r} starts at {lo}, the data before it ends at {at}")
        at = hi
    if at != data_len:
        raise ValueError(f"safetensors header: the tensors cover {at} bytes of a {data_len}-byte data region")
    return extra, entries


def _check_into(into: Mapping, entries, ctx, sliced: bool = False, stored: Mapping | None = None) -> None:
    """Every mismatch between ``into`` and the header's tensors (``sliced``: the selected slices, for
    ``read_safetensors_slices``), in one ``ValueError``.  ``stored``: {name: the file's dtype} of the tensors that are
    converted to the dtype ``entries`` gives them."""
    problems = []
    want = {name: (dtype, shape) for name, dtype, shape, _, _ in entries}
    stored = stored or {}
    there, what, holds = ("selected", "read_safetensors_slices", "the slice is") if sliced else \
        ("in the file", "read_safetensors", "the file holds")
    for name in sorted(set(want) - set(into)):
        problems.append(f"{name!r} is {there} but not in into")
    for name in sorted(set(into) - set(want)):
        problems.append(f"{name!r} is in into but not {there}")
    spans = []
    for name in sorted(set(want) & set(into)):
        t, (dtype, shape) = into[name], want[name]
        if t.dtype != dtype or list(t.shape) != shape:
            if name in stored:
                problems.append(f"{name!r}: {holds} {stored[name]} {shape}, converted to {dtype}, into has {t.dtype} "
                                f"{list(t.shape)}")
            else:
                problems.append(f"{name!r}: {holds} {dtype} {shape}, into has {t.dtype} {list(t.shape)}")
            continue
        try:
            DeviceFile._Source._check_tensor(t, ctx, f"into[{name!r}]")
        except ValueError as exc:
            problems.append(str(exc))
            continue
        if t.numel():
            spans.append((t.data_ptr(), t.data_ptr() + t.numel() * t.element_size(), name))
    spans.sort()
    for (_, hi, a), (lo, _, b) in zip(spans, spans[1:]):
        if lo < hi:
            problems.append(f"into[{a!r}] and into[{b!r}] overlap")
    if problems:
        raise ValueError(f"{what}(into=...): " + "; ".join(problems))


async def _load_runs(client, volume_id: str, files, staging_bytes: int) -> None:
    """Load ``files`` -- ``(path, runs, dst, start, end)`` each, ``runs`` ``[((F, W, P, R) as _slice_runs gives it,
    packed offset in dst, (stored dtype, target dtype), (FP8 dtype, target dtype, _Dequant) or None)]`` -- into their
    ``dst``: ONE ``VolumeGetFile2`` call per file that has a touched block, over its bytes [start, end), all made
    concurrently, then exactly the blocks that hold a byte of a run, once each, into the page-locked waves of ONE
    ``_load_in_waves``, so a wave may hold the blocks of several files.  Each complete wave makes at most one
    ``load_boxes`` call (the unconverted runs; one also when nothing converts), at most one ``load_cast_boxes`` call,
    at most one ``load_scaled_boxes`` call (the dequantized runs), and for the runs of weights quantized to FP8 (a
    ``_Quant``) at most one ``load_fp8_amax_boxes`` call (every box of the wave) and one ``load_quant_boxes`` call (the
    bands the wave completes, with the boxes of their first part that landed in the previous wave, whose half is then
    not refilled before this copy has read it), all on one stream, over every file's ``dst``:
    every run is cut into boxes, split where the staging stops being contiguous, at a wave's edge, a skipped block or
    the next file.  A converted run's packed offsets count target bytes."""
    BS = blob_utils.BLOCK_SIZE
    touched = [_touched_blocks([r for r, _, _ in runs], BS) for _, runs, _, _, _ in files]
    live = [files[k] for k, t in enumerate(touched) if t]
    touched = [t for t in touched if t]
    if not live:
        return
    answers = await gather_cancel_on_error(*[_block_slices(client, volume_id, path, start, end - start)
                                             for path, _, _, start, end in live])
    slices = [(url, off, m, i) for i, ((_, _, _, start, _), got) in enumerate(zip(live, answers))
              for url, off, m in got if (start + off) // BS in touched[i]]
    dsts = [dst for _, _, dst, _, _ in live]

    def load(wave, at, buf, ctx):
        plain, cast, scaled, k = [], [], [], 0
        landed = {}  # _Quant -> [(file offset, end, staging offset, file, weight's packed offset)] of this wave
        while k < len(wave):  # a stretch: blocks of one file, adjacent in the file and in the buffer
            e, i = k + 1, wave[k][3]
            while e < len(wave) and wave[e][3] == i and wave[e][1] == wave[e - 1][1] + wave[e - 1][2] and \
                    at[e] == at[e - 1] + wave[e - 1][2]:
                e += 1
            _, runs, _, start, _ = live[i]
            s0, s1 = start + wave[k][1], start + wave[e - 1][1] + wave[e - 1][2]
            for run, d, conv in runs:
                for b in _clip_run(run, 0, s0, s1, at[k]):
                    if conv is None:
                        plain.append((i, d + b[0], *b[1:]))
                    elif len(conv) == 2:  # the box's offset in the run, in source bytes, to target bytes
                        cast.append((i, d + b[0] // conv[0].itemsize * conv[1].itemsize, *b[1:], *conv))
                    elif isinstance(conv[2], _Quant):  # a whole weight's run: one row per box
                        lo = s0 + b[3] - at[k]
                        landed.setdefault(conv[2], []).append((lo, lo + b[1], b[3], i, d))
                    else:  # one-byte elements; the box's first element in the weight, from its file offset
                        q = conv[2]
                        scaled.append((i, d + b[0] * conv[1].itemsize, *b[1:], conv[0], conv[1], q.scales,
                                       s0 + b[3] - at[k] - q.start, q.rows, q.cols, q.block_rows, q.block_cols))
            k = e
        amax, quant, bands, carried = [], [], [], False
        for q, now in landed.items():  # every box's amax; then the bands this wave completes, their carried part too
            amax += [q.box(*x) for x in now]
            top = max(hi for _, hi, *_ in now)
            done = q.nbands if top == q.end else (top - q.start) // q.band
            edge = min(q.start + done * q.band, q.end)
            if done > q.done:
                quant += [q.box(*x) for x in _clip_landed(q.pending + now, q.start + q.done * q.band, edge)]
                bands.append((q.amax, q.scales, q.done * q.grid_cols, (done - q.done) * q.grid_cols))
                carried = carried or bool(q.pending)
                q.done = done
            q.pending = _clip_landed(q.pending + now, edge, q.end)
        loaded = load_boxes(dsts, plain, buf, ctx=ctx) if plain or not (cast or scaled or amax) else None
        if cast:  # on the same stream as the plain boxes: its completion implies theirs
            loaded = load_cast_boxes(dsts, cast, buf, ctx=ctx)
        if scaled:  # the same stream again
            loaded = load_scaled_boxes(dsts, scaled, buf, ctx=ctx)
        if amax:  # the same stream: the amax of a wave is in before its bands are finalized
            loaded = load_fp8_amax_boxes(dsts, amax, buf, ctx=ctx)
        if bands:
            loaded = load_quant_boxes(dsts, quant, bands, buf, ctx=ctx)
        return (loaded, True) if carried else loaded

    await _load_in_waves(slices, load, staging_bytes, None, lambda **_: None)


async def read_safetensors(client, volume_id: str, path: str, *, into: Mapping | None = None, dtype=None,
                           scales: Mapping | None = None, scale_block=(128, 128), fp8=None,
                           scale_suffix: str = "_scale_inv", staging_bytes: int = 256 << 20) -> dict:
    """The safetensors file at ``path`` as ``{name: tensor}`` on the context's device, equal to what
    ``safetensors.torch.load`` gives for the file's bytes (same names, dtypes, shapes and values; keys in data order).

    The 8-byte header length and the header come through host memory (two small ranged reads) and are checked as the
    safetensors library checks them, ``ValueError`` before any tensor is allocated.  The tensors are ``torch.empty`` on
    the context's device, or with ``into=`` the caller's tensors, filled in place: names, dtypes and shapes must match
    exactly and the tensors must be contiguous, on the context's device and not overlap; every mismatch is listed in one
    ``ValueError`` before any block GET.  The data region then arrives with one ``read_file_into_device`` into a
    ``DeviceFile`` over the tensors in data order (``staging_bytes`` as there).

    ``dtype`` converts tensors as they land, each result equal bit for bit to ``full.to(dtype)`` on the device: a torch
    dtype (float32, float16 or bfloat16) for every F32 / F16 / BF16 tensor, integer and bool tensors unchanged, or
    ``{name: dtype}`` for the tensors it names.  ``cast_targets`` lists what it refuses, in one ``ValueError`` before
    any data GET (a file not written by ``safetensors.torch.save`` may hold a tensor that cannot convert in place).
    With ``into=`` each tensor must have its target dtype.  When something converts, the same ``VolumeGetFile2`` call
    and block GETs as without ``dtype`` feed the waves of ``_load_runs``: HBM holds only the results, never the stored
    image; when nothing converts, the call is the one without ``dtype``.

    ``scales={weight: scale name}`` (``fp8_scales`` pairs them by name) dequantizes FP8 weights (F8_E4M3, F8_E5M2;
    2-D, R x C) as they land, to their target from ``dtype`` (the single dtype, or the weight's entry of a mapping; a
    single dtype still refuses FP8 tensors without a scale).  The scale S (F32, F16 or BF16) holds one value per
    ``scale_block`` = (rows, columns) block, ``None`` meaning the whole dimension: shape [ceil(R / rows), ceil(C /
    columns)] ([] or [1] for one block, [ceil(R / rows)] for one block column).  Each result equals, bit for bit, what
    torch computes on CUDA: ``(W.float() * S.float().repeat_interleave(rows, 0)[:R].repeat_interleave(columns,
    1)[:, :C]).to(target)``.  Scale tensors are consumed: not in the result, and not allowed in ``into``.
    ``_scale_targets`` lists every problem in one ``ValueError`` before any data GET.  The scales load first into
    temporary tensors (one ``_load_runs`` over their blocks), then everything else (a second one, whose waves make at
    most one ``load_boxes``, one ``load_cast_boxes`` and one ``load_scaled_boxes`` call); HBM holds the results and the
    scales, never the FP8 image, and the scales are freed on return.

    ``fp8=names`` quantizes the named weights (non-empty 2-D F32 / F16 / BF16 tensors) to ``torch.float8_e4m3fn`` as
    they land, in ``scale_block`` blocks as above, and returns each one's F32 scale tensor ([ceil(R / rows),
    ceil(C / columns)]) as ``name + scale_suffix``, right after the weight: both bit for bit what
    ``DeviceFile.safetensors({...}, fp8=names, scale_block=..., scale_suffix=...)`` stores for it (DESIGN §5.20).
    Every other tensor is read as without ``fp8``, converted by ``dtype`` if given.  With ``into=`` a weight needs a
    contiguous float8_e4m3fn tensor of its shape and its scale name an F32 tensor of the grid's shape.  The blocks,
    the requests and the waves are those of a read with ``dtype``; each wave reduces the amax of the weights' boxes
    into one temporary F32 array (one value per block), then finalizes and quantizes every band (the block_rows rows of
    one block row) whose last byte has landed, so HBM holds only the results, their scales and that array.  A band must
    touch at most ``staging_bytes // 2 // BLOCK_SIZE + 1`` blocks.  ``fp8`` with ``scales``, a name that is not such a
    weight or is given twice, a name a ``dtype`` mapping names, a scale name that is already a tensor and a band too
    large for ``staging_bytes`` are refused, every problem in one ``ValueError`` before any data GET."""
    ctx = blob_utils.get_context()
    size, n, _, entries = await _read_safetensors_header(client, volume_id, path)
    if scales or fp8 is not None:
        if staging_bytes < 2 * blob_utils.BLOCK_SIZE:
            raise ValueError(f"staging_bytes must hold two blocks ({2 * blob_utils.BLOCK_SIZE} bytes), got "
                             f"{staging_bytes}")
        return await _read_shards(client, volume_id, path, [(path, n, entries)], None, into, dtype, scales,
                                  scale_block, staging_bytes, ctx, fp8, scale_suffix)
    targets = cast_targets(path, dtype, entries, 8 + n)
    if targets and staging_bytes < 2 * blob_utils.BLOCK_SIZE:
        raise ValueError(f"staging_bytes must hold two blocks ({2 * blob_utils.BLOCK_SIZE} bytes), got {staging_bytes}")
    result = [(name, targets.get(name, dt), shape, lo, hi) for name, dt, shape, lo, hi in entries]
    if into is not None:
        _check_into(into, result, ctx, stored={name: dt for name, dt, *_ in entries if name in targets})
        tensors = [into[name] for name, *_ in entries]
    else:
        tensors = [DeviceFile._Source._new_tensor(shape, dt, ctx) for _, dt, shape, _, _ in result]
    if entries and size - 8 - n:
        dst = DeviceFile._over(DeviceFile._Source(tensors, BOUNCE_BYTES))
        if not targets:
            await read_file_into_device(client, volume_id, path, dst, start=8 + n, staging_bytes=staging_bytes)
        else:
            runs, dest = [], 0
            for (name, dt, _, lo, hi), t in zip(entries, tensors):
                if hi > lo:
                    runs.append(((8 + n + lo, hi - lo, hi - lo, 1), dest, (dt, t.dtype) if name in targets else None))
                dest += t.numel() * t.element_size()
            await _load_runs(client, volume_id, [(path, runs, dst, 8 + n, size)], staging_bytes)
    return {name: t for (name, *_), t in zip(entries, tensors)}


_ST_MAX_HEADER = 100_000_000  # the safetensors library's bound on the header length


async def _read_safetensors_header(client, volume_id: str, path: str):
    """(file size, header length, ``__metadata__`` or None, ``_safetensors_entries``) of the safetensors file at
    ``path``: three ``VolumeGetFile2`` calls (the size, then the 8-byte length and the header through host memory)."""
    size = (await _get_file2(client, volume_id, path, 0, 8)).size
    if size < 8:
        raise ValueError(f"{path} ({size} bytes) is too short to be a safetensors file")
    n = int.from_bytes(await _read_range_host(client, volume_id, path, 0, 8), "little")
    if n > _ST_MAX_HEADER:
        raise ValueError(f"safetensors header of {n} bytes is larger than {_ST_MAX_HEADER}")
    if 8 + n > size:
        raise ValueError(f"safetensors header of {n} bytes does not fit a {size}-byte file")
    metadata, entries = _safetensors_entries(await _read_range_host(client, volume_id, path, 8, n), size - 8 - n)
    return size, n, metadata, entries


async def read_safetensors_header(client, volume_id: str, path: str):
    """(``__metadata__`` or None, {name: (torch dtype, shape tuple)} in data order) of the safetensors file at
    ``path``, read and checked as ``read_safetensors`` reads its header (three ``VolumeGetFile2`` calls, no data): what
    a caller needs to work out its slices for ``read_safetensors_slices``."""
    _, _, metadata, entries = await _read_safetensors_header(client, volume_id, path)
    return metadata, {name: (dtype, tuple(shape)) for name, dtype, shape, _, _ in entries}


def _slice_bounds(name: str, shape, index):
    """([(lo, hi) per dimension], kept: [bool per dimension]) of ``full[index]`` for a tensor of ``shape``: ``index``
    an int, a slice of step 1, ``...`` or a tuple of these.  ``TypeError`` / ``ValueError`` / ``IndexError`` as the
    class of the problem, as torch raises them."""
    items = index if isinstance(index, tuple) else (index,)
    for x in items:
        if x is Ellipsis:
            continue
        if isinstance(x, bool) or not isinstance(x, (int, slice)):
            raise TypeError(f"{name!r}: index {x!r} is not an int, a slice or ...; only those are supported")
        if isinstance(x, slice):
            if x.step not in (None, 1):
                raise ValueError(f"{name!r}: slice {x!r} has a step other than 1")
            for v in (x.start, x.stop):
                if v is not None and (isinstance(v, bool) or not isinstance(v, int)):
                    raise TypeError(f"{name!r}: slice {x!r} has a bound that is not an int or None")
    ellipses = sum(x is Ellipsis for x in items)
    if ellipses > 1:
        raise IndexError(f"{name!r}: an index can only have a single ellipsis ('...')")
    rank = len(shape)
    if len(items) - ellipses > rank:
        raise IndexError(f"{name!r}: too many indices for tensor of dimension {rank}")
    if ellipses:
        at = next(i for i, x in enumerate(items) if x is Ellipsis)
        items = items[:at] + (slice(None),) * (rank - len(items) + 1) + items[at + 1 :]
    items = items + (slice(None),) * (rank - len(items))
    bounds, kept = [], []
    for dim, (x, d) in enumerate(zip(items, shape)):
        if isinstance(x, slice):
            lo, hi, _ = x.indices(d)
            bounds.append((lo, max(lo, hi)))
            kept.append(True)
        else:
            if not -d <= x < d:
                raise IndexError(f"{name!r}: index {x} is out of bounds for dimension {dim} with size {d}")
            bounds.append((x % d, x % d + 1))
            kept.append(False)
    return bounds, kept


def _slice_runs(shape, bounds, itemsize: int, start: int):
    """The selection ``bounds`` of a C-contiguous tensor at file offset ``start``, as patterns ``(F, W, P, R)``: R rows
    of W bytes, row r at file offset F + r * P (P >= W), in the order their bytes are packed into the result.  The
    trailing whole dimensions merge into the row width; the dimensions out to the next partial one, which must be whole
    but for the outermost, make the rows at one pitch; the dimensions outside that are enumerated."""
    import itertools

    if any(hi == lo for lo, hi in bounds):
        return []
    rank = len(shape)
    whole = [lo == 0 and hi == d for (lo, hi), d in zip(bounds, shape)]
    stride = [itemsize] * (rank + 1)  # stride[j]: bytes per index step of dimension j (stride[rank] = one element)
    for j in range(rank - 1, -1, -1):
        stride[j] = stride[j + 1] * shape[j]
    k = max((j for j in range(rank) if not whole[j]), default=-1)
    if k < 0:  # the whole tensor (a 0-d tensor included)
        return [(start, stride[0] if rank else itemsize, stride[0] if rank else itemsize, 1)]
    width = (bounds[k][1] - bounds[k][0]) * stride[k + 1]
    m = max((j for j in range(k) if not whole[j]), default=-1)  # the rows run over dimensions max(m, 0) .. k - 1
    rows = 1
    for j in range(max(m, 0), k):
        rows *= bounds[j][1] - bounds[j][0]
    pitch = stride[k] if k else width
    base = start + bounds[k][0] * stride[k + 1] + (bounds[m][0] * stride[m + 1] if m >= 0 else 0)
    return [(base + sum(i * stride[j + 1] for j, i in enumerate(combo)), width, pitch, rows)
            for combo in itertools.product(*[range(lo, hi) for lo, hi in bounds[: max(m, 0)]])]


def _touched_blocks(runs, BS: int) -> set:
    """The blocks (file offset // BS) that hold a byte of a row of ``runs``."""
    out = set()
    for F, W, P, R in runs:
        if R == 1 or P - W < BS:  # no block fits between two rows: every block of the span is touched
            out.update(range(F // BS, (F + (R - 1) * P + W - 1) // BS + 1))
        else:
            for r in range(R):
                out.update(range((F + r * P) // BS, (F + r * P + W - 1) // BS + 1))
    return out


def _clip_run(run, dest: int, s0: int, s1: int, at: int):
    """The boxes ``(dest offset, width, rows, staging offset, pitch)`` of the bytes of ``run`` (packed from ``dest``)
    that lie in file bytes [s0, s1), staged contiguously from buffer offset ``at``: a partial first row, the whole
    rows at the run's pitch, a partial last row."""
    F, W, P, R = run
    if F >= s1 or F + (R - 1) * P + W <= s0:
        return []
    ra = 0 if s0 <= F else max(0, (s0 - F - W) // P + 1)  # the first row that ends after s0
    rb = min(R - 1, (s1 - F - 1) // P)  # the last row that starts before s1
    if ra > rb:
        return []

    def part(r):
        c0, c1 = max(0, s0 - F - r * P), min(W, s1 - F - r * P)
        return (dest + r * W + c0, c1 - c0, 1, at + F + r * P + c0 - s0, c1 - c0)

    if ra == rb:
        return [part(ra)]
    out, tail = [], []
    if F + ra * P < s0:
        out.append(part(ra))
        ra += 1
    if F + rb * P + W > s1:
        tail.append(part(rb))
        rb -= 1
    if ra <= rb:
        out.append((dest + ra * W, W, rb - ra + 1, at + F + ra * P - s0, P))
    return out + tail


async def read_safetensors_slices(client, volume_id: str, path: str, select: Mapping, *, into: Mapping | None = None,
                                  dtype=None, scales: Mapping | None = None, scale_block=(128, 128),
                                  staging_bytes: int = 256 << 20) -> dict:
    """Slices of tensors of the safetensors file at ``path``: ``{name: full[index]}`` for every ``name: index`` of
    ``select``, in its order, each a new contiguous tensor on the context's device (``full`` as ``read_safetensors``
    returns it; for these index forms also what ``safe_open(...).get_slice(name)[index]`` gives).  An index is an int
    (negative allowed), a slice of step 1 (bounds clamped as Python clamps them), at most one ``...``, or a tuple of
    these no longer than the tensor's rank; ``...`` or ``()`` is the whole tensor.  Anything else raises before any data
    GET: ``TypeError`` for ``None``, lists, tensors and bools, ``ValueError`` for other steps, ``IndexError`` for an
    out-of-range int or too many indices, and one ``ValueError`` naming every unknown name.

    The header is read as ``read_safetensors`` reads it.  Then ONE ``VolumeGetFile2`` call covers the first touched
    block to the last touched byte, and exactly the touched blocks (those holding a selected byte) are fetched, once
    each, into the page-locked waves of ``read_file_into_device`` (``staging_bytes`` as there).  Each complete wave
    goes to the device with one ``load_boxes`` call: every selection is cut into boxes (rows at one pitch, the trailing
    whole dimensions merged into the row), split where the staging stops being contiguous, at a wave's edge or a
    skipped block.  Of HBM, the call allocates only the results and the copy's small stream-ordered tables.  With ``into=`` the caller's tensors are filled
    in place: the sliced shapes and the dtypes must match, and the tensors must be contiguous, on the context's device
    and not overlap, every mismatch in one ``ValueError`` before any data GET.  On return and on error, ordering and
    partial content are as for ``read_safetensors``.  ``dtype`` converts the slices as they land, as
    ``read_safetensors`` does (a mapping names selected tensors); each result equals ``full[index].to(dtype)`` bit for
    bit, and the requests are those of the call without ``dtype``.  ``scales`` and ``scale_block`` dequantize FP8
    weights as ``read_safetensors`` does; every weight named in ``scales`` must be selected and its scale must not be.
    A slice takes the scale of each element's place in the full tensor, so it equals ``dequantized_full[index]``."""
    BS = blob_utils.BLOCK_SIZE
    if staging_bytes < 2 * BS:
        raise ValueError(f"staging_bytes must hold two blocks ({2 * BS} bytes), got {staging_bytes}")
    ctx = blob_utils.get_context()
    _, n, _, entries = await _read_safetensors_header(client, volume_id, path)
    if scales:
        return await _read_shards(client, volume_id, path, [(path, n, entries)], select, into, dtype, scales,
                                  scale_block, staging_bytes, ctx)
    by_name = {e[0]: e for e in entries}
    unknown = [name for name in select if name not in by_name]
    if unknown:
        raise ValueError(f"{path}: no tensors named {', '.join(repr(u) for u in unknown)}")
    plans = []  # (name, dtype, result shape, runs)
    for name, index in select.items():
        _, dt, shape, lo, _ = by_name[name]
        bounds, kept = _slice_bounds(name, shape, index)
        result = [hi - b for (b, hi), k in zip(bounds, kept) if k]
        plans.append((name, dt, result, _slice_runs(shape, bounds, dt.itemsize, 8 + n + lo)))
    targets = cast_targets(path, dtype, [by_name[name] for name in select], 8 + n, sliced=True)
    if into is not None:
        _check_into(into, [(name, targets.get(name, dt), result, 0, 0) for name, dt, result, _ in plans], ctx,
                    sliced=True, stored={name: dt for name, dt, *_ in plans if name in targets})
        tensors = [into[name] for name, *_ in plans]
    else:
        tensors = [DeviceFile._Source._new_tensor(result, targets.get(name, dt), ctx) for name, dt, result, _ in plans]
    runs, base = [], 0  # (run, its packed offset in the one file over every result tensor, conversion)
    for (name, dt, _, rs), t in zip(plans, tensors):
        dest, conv = base, (dt, t.dtype) if name in targets else None
        for run in rs:
            runs.append((run, dest, conv))
            dest += run[1] * run[3] // dt.itemsize * t.element_size()
        base += t.numel() * t.element_size()
    if runs:
        first = min(_touched_blocks([r for r, _, _ in runs], BS)) * BS
        end = max(F + (R - 1) * P + W for (F, W, P, R), _, _ in runs)
        dst = DeviceFile._over(DeviceFile._Source(tensors, BOUNCE_BYTES))
        await _load_runs(client, volume_id, [(path, runs, dst, first, end)], staging_bytes)
    return {name: t for (name, *_), t in zip(plans, tensors)}


async def _read_index(client, volume_id: str, index_path: str):
    """(index metadata or None, [(shard path, header length, entries)] in shard order) of the sharded safetensors
    checkpoint whose ``model.safetensors.index.json`` is at ``index_path``: the index through host memory (one
    ``VolumeGetFile2`` call), then every shard's header concurrently (three each, as ``read_safetensors`` reads one).
    The shards are the index's file names, sorted, each relative to the index's directory; every disagreement between
    ``weight_map`` and the shards' headers is listed in one ``ValueError`` before any data GET."""
    raw = b"".join([body async for body in read_file(client, volume_id, index_path)])
    try:
        index = json.loads(raw.decode("utf-8"))
    except (UnicodeDecodeError, ValueError) as exc:
        raise ValueError(f"{index_path} is not a valid JSON index: {exc}") from None
    weight_map = index.get("weight_map") if isinstance(index, dict) else None
    if not isinstance(weight_map, dict) or not all(isinstance(v, str) for v in weight_map.values()):
        raise ValueError(f"{index_path}: the index needs a weight_map of tensor name -> shard file name")
    names = sorted(set(weight_map.values()))
    bad = [f for f in names if not f or PurePosixPath(f).is_absolute() or ".." in PurePosixPath(f).parts]
    if bad:
        raise ValueError(f"{index_path}: shard names must be relative to the index's directory without '..': "
                         f"{', '.join(map(repr, bad))}")
    base = PurePosixPath(index_path).parent
    paths = [(base / f).as_posix() for f in names]
    headers = await gather_cancel_on_error(*[_read_safetensors_header(client, volume_id, p) for p in paths])
    problems, holder = [], {}
    for f, (_, _, _, entries) in zip(names, headers):
        held = {e[0] for e in entries}
        for name in held:
            if name in holder:
                problems.append(f"{name!r} is in both {holder[name]} and {f}")
            holder.setdefault(name, f)
            if name not in weight_map:
                problems.append(f"{f} holds {name!r}, which weight_map does not name")
            elif weight_map[name] != f:
                problems.append(f"{f} holds {name!r}, which weight_map maps to {weight_map[name]}")
    held_by = {f: {e[0] for e in h[3]} for f, h in zip(names, headers)}
    for name, f in weight_map.items():
        if name not in held_by[f]:
            problems.append(f"weight_map maps {name!r} to {f}, which does not hold it")
    if problems:
        raise ValueError(f"{index_path}: " + "; ".join(sorted(problems)))
    metadata = index.get("metadata")
    return metadata, [(p, n, entries) for p, (_, n, _, entries) in zip(paths, headers)]


async def read_safetensors_index(client, volume_id: str, index_path: str):
    """(the index's ``metadata``, {name: (shard path, torch dtype, shape tuple)} in shard order, then data order) of
    the sharded safetensors checkpoint whose index (``model.safetensors.index.json``) is at ``index_path``: the index
    through host memory, then every shard's header, concurrently.  Shard names are resolved against the index's
    directory; absolute names and names with ``..`` are refused.  A name of ``weight_map`` that its shard does not hold,
    a tensor a shard holds that ``weight_map`` maps elsewhere (or not at all), and a name two shards hold are all
    reported in one ``ValueError``, before any data GET."""
    metadata, shards = await _read_index(client, volume_id, index_path)
    return metadata, {name: (path, dtype, tuple(shape)) for path, _, entries in shards
                      for name, dtype, shape, _, _ in entries}


async def read_safetensors_sharded(client, volume_id: str, index_path: str, *, select: Mapping | None = None,
                                   into: Mapping | None = None, dtype=None, scales: Mapping | None = None,
                                   scale_block=(128, 128), fp8=None, scale_suffix: str = "_scale_inv",
                                   staging_bytes: int = 256 << 20) -> dict:
    """A sharded safetensors checkpoint (the index at ``index_path``, read as ``read_safetensors_index`` reads it) as
    ``{name: tensor}`` on the context's device: what merging ``read_safetensors`` over every shard returns, keys in
    shard order, then data order.  With ``select={name: index}`` it is what ``read_safetensors_slices`` returns for
    those names instead, in ``select``'s order.  ``into=``, ``dtype=``, ``scales=`` and ``scale_block=`` mean what
    they mean there, with the same messages, every problem in one ``ValueError`` before any data GET; a weight and its
    scale may live in different shards.

    Every shard's data comes through one wave loop: ONE ``VolumeGetFile2`` call per shard with a touched byte, all
    made concurrently, then every touched block once (untouched blocks of a selection never), the blocks of all shards
    in one sequence of page-locked waves (``staging_bytes`` as in ``read_file_into_device``), so a wave may hold blocks
    of several shards and the pipeline does not drain between shards.  Each complete wave makes at most one
    ``load_boxes`` and one ``load_cast_boxes`` call (and with ``scales=`` one ``load_scaled_boxes`` call), over a
    ``DeviceFile`` per shard.  Of HBM, the call allocates only the results and the copies' small tables (and with
    ``scales=`` the scales, freed on return).  Ordering and partial content on return and on error are as for
    ``read_safetensors``.  ``fp8=`` and ``scale_suffix=`` quantize weights as ``read_safetensors`` does, each scale
    right after its weight; a band never spans shards, and each wave adds at most one ``load_fp8_amax_boxes`` and one
    ``load_quant_boxes`` call."""
    BS = blob_utils.BLOCK_SIZE
    if staging_bytes < 2 * BS:
        raise ValueError(f"staging_bytes must hold two blocks ({2 * BS} bytes), got {staging_bytes}")
    ctx = blob_utils.get_context()
    _, shards = await _read_index(client, volume_id, index_path)
    return await _read_shards(client, volume_id, index_path, shards, select, into, dtype, scales, scale_block,
                              staging_bytes, ctx, fp8, scale_suffix)


class _Dequant:
    """How the boxes of one FP8 weight are dequantized: its scales on the device, the file offset of its element 0,
    its shape and its block (a block of the whole dimension is the dimension)."""

    def __init__(self, scales, start: int, rows: int, cols: int, block_rows: int, block_cols: int):
        self.scales, self.start, self.rows, self.cols = scales, start, rows, cols
        self.block_rows, self.block_cols = block_rows, block_cols


class _Quant:
    """How the boxes of one weight are quantized to FP8 E4M3 as they land: its a (``amax``, a view of the read's one
    amax array) and its result ``scales``, the file offset of its element 0, its shape, its block (a block of the whole
    dimension is the dimension) and its source element size.  A band -- the block_rows rows of one block row, one
    contiguous byte range of the file -- is quantized once all of it has landed: ``done`` bands are so far, and
    ``pending`` holds the landed boxes of the next one (``(file offset, end, staging offset, file, weight's packed
    offset)``), which all lie in the previous wave's half."""

    def __init__(self, amax, scales, start: int, rows: int, cols: int, block_rows: int, block_cols: int,
                 src_dtype):
        self.amax, self.scales, self.start, self.rows, self.cols = amax, scales, start, rows, cols
        self.block_rows, self.block_cols, self.src_dtype = block_rows, block_cols, src_dtype
        self.itemsize = src_dtype.itemsize
        self.end, self.band = start + rows * cols * self.itemsize, block_rows * cols * self.itemsize
        self.nbands, self.grid_cols = -(-rows // block_rows), -(-cols // block_cols)
        self.done, self.pending = 0, []

    def box(self, lo: int, hi: int, at: int, i: int, d: int):
        """The ``load_fp8_amax_boxes`` / ``load_quant_boxes`` box of file bytes [lo, hi) staged at ``at``."""
        e = (lo - self.start) // self.itemsize
        return (i, d + e, hi - lo, 1, at, hi - lo, self.src_dtype, self.amax, e, self.rows, self.cols,
                self.block_rows, self.block_cols)


def _clip_landed(boxes, lo: int, hi: int) -> list:
    """The parts of ``_Quant`` landed boxes that lie in file bytes [lo, hi)."""
    return [(max(a, lo), min(b, hi), at + max(a, lo) - a, i, d) for a, b, at, i, d in boxes if max(a, lo) < min(b, hi)]


def _band_blocks(start: int, rows: int, cols: int, block_rows: int, itemsize: int, BS: int) -> int:
    """The most staging blocks one band of a weight (file offset ``start``) touches."""
    band, end = block_rows * cols * itemsize, start + rows * cols * itemsize
    lo = start + band * np.arange(-(-rows // block_rows), dtype=np.int64)
    hi = np.minimum(lo + band, end)
    return int(((hi - 1) // BS - lo // BS + 1).max())


def _fp8_load_plan(there: str, tensors: Mapping, starts: Mapping, fp8, scale_block, scale_suffix, dtype, scales,
                   select, staging_bytes: int, problems: list) -> dict:
    """{weight: scale name}, in the order of ``tensors`` ({name: (torch dtype, shape)}, ``there`` names where they are;
    ``starts``: their file offsets),
    of the weights ``fp8`` quantizes on load; every problem is appended to ``problems``: ``scales`` or ``select`` given
    too, a bad ``scale_block`` or ``scale_suffix``, unknown or repeated names, weights that are not non-empty 2-D
    F32 / F16 / BF16 tensors, a name that a ``dtype`` mapping names too, a scale name that is already a tensor, and a
    weight whose band touches more staging blocks than a wave can carry into the next (``per_half + 1``)."""
    if scales:
        problems.append("fp8 cannot be combined with scales (the FP8 weights of a file are dequantized, not quantized)")
    if select is not None:
        problems.append("fp8 does not take select= (slices are not quantized on load)")
    if isinstance(fp8, str):
        fp8 = None  # a single name is a common slip: refused, not read as its characters
    try:
        names = list(fp8)
    except TypeError:
        problems.append("fp8 must be an iterable of tensor names")
        return {}
    good_block = isinstance(scale_block, (tuple, list)) and len(scale_block) == 2 and all(
        b is None or (isinstance(b, int) and not isinstance(b, bool) and b >= 1) for b in scale_block)
    if not good_block:
        problems.append(f"scale_block {scale_block!r} must be (rows, columns), each an int >= 1 or None (the whole "
                        f"dimension)")
    if not isinstance(scale_suffix, str):
        problems.append(f"scale_suffix must be a str, got {scale_suffix!r}")
        scale_suffix = None
    want, codes = set(), cast_dtypes()
    for n in names:
        if n in want:
            problems.append(f"{n!r} is in fp8 twice")
        elif not isinstance(n, str) or n not in tensors:
            problems.append(f"{n!r} is in fp8 but not {there}")
        else:
            want.add(n)
    BS = blob_utils.BLOCK_SIZE
    per_half = staging_bytes // 2 // BS
    plan = {}
    for n, (dt, shape) in tensors.items():
        if n not in want:
            continue
        if len(shape) != 2 or 0 in shape:
            problems.append(f"{n!r} has shape {list(shape)}; fp8 quantizes non-empty 2-D weights")
        elif dt not in codes:
            problems.append(f"{n!r} is {_st_dtypes()[dt][0]}; only F32, F16 and BF16 weights quantize")
        elif good_block:
            R, C = shape
            br = min(R, scale_block[0] or R)
            need = _band_blocks(starts[n], R, C, br, dt.itemsize, BS)
            if need > per_half + 1:
                problems.append(f"{n!r}: one band of {br} rows ({br * C * dt.itemsize} bytes) touches {need} staging "
                                f"blocks, and staging_bytes={staging_bytes} carries {per_half + 1}; "
                                f"staging_bytes={2 * max(1, need - 1) * BS} would hold it")
        if isinstance(dtype, Mapping) and n in dtype:
            problems.append(f"{n!r} is in both fp8 and dtype")
        if scale_suffix is not None:
            if n + scale_suffix in tensors:
                problems.append(f"the scale of {n!r}, {n + scale_suffix!r}, is already a tensor of the checkpoint")
            plan[n] = n + scale_suffix
    return plan


def _scale_grid(shape, scale_block):
    """(scale rows, scale columns) of a 2-D weight of ``shape`` in blocks ``scale_block`` (None: the whole dimension)."""
    return tuple(1 if b is None else -(-d // b) for d, b in zip(shape, scale_block))


def fp8_scales(names, suffix: str = "_scale_inv") -> dict:
    """``{weight: scale}`` for every name ``n`` of ``names`` for which ``n + suffix`` is a name too, in the order of
    ``names``: the ``scales=`` argument of the ``read_safetensors*`` calls.  ``names`` may be the tensors of
    ``read_safetensors_header`` or of ``read_safetensors_index``.  DeepSeek-V3/R1 and the Qwen3 FP8 checkpoints store
    ``<weight>_scale_inv`` (the default); compressed-tensors checkpoints store ``<weight>_scale``."""
    names = list(names)
    have = set(names)
    return {n: n + suffix for n in names if n + suffix in have}


def _scale_targets(where: str, there: str, dtype, scales: Mapping, scale_block, tensors: Mapping, select, into) -> dict:
    """{weight: target dtype} of the FP8 weights of ``scales`` ({weight: scale name}), whose tensors ``tensors`` gives
    as {name: (torch dtype, shape)} (``there`` names where they are).  Every problem in one ``ValueError``: ``scales``
    without ``dtype``, a bad ``scale_block``, unknown or unselected weights, missing scales, a weight that is not FP8 or
    not 2-D, a scale that is not F32 / F16 / BF16 or has the wrong shape for the block, a name that is both a weight
    and a scale, a scale that is selected or in ``into``, and a missing or unsupported target."""
    import torch

    if not isinstance(scales, Mapping):
        raise ValueError(f"{where}: scales must map weight names to scale names, got {type(scales).__name__}")
    codes, fp8, tags = cast_dtypes(), fp8_dtypes(), _st_dtypes()
    supported = "float32, float16 or bfloat16"
    problems = []
    if dtype is None:
        problems.append("scales needs dtype= (the dtype the weights are dequantized to)")
    good_block = isinstance(scale_block, (tuple, list)) and len(scale_block) == 2 and all(
        b is None or (isinstance(b, int) and not isinstance(b, bool) and b >= 1) for b in scale_block)
    if not good_block:
        problems.append(f"scale_block {scale_block!r} is not a pair of ints >= 1 or None")
    for name in sorted(set(scales) & set(scales.values())):
        problems.append(f"{name!r} is both a weight and a scale")
    if isinstance(dtype, Mapping):
        for name in sorted(set(dtype) & set(scales.values())):
            problems.append(f"{name!r} is a scale, which is consumed, but dtype names it")
    out = {}
    for w, sc in scales.items():
        if w not in tensors:
            problems.append(f"weight {w!r} is not {there}")
        elif select is not None and w not in select:
            problems.append(f"weight {w!r} is not selected")
        elif tensors[w][0] not in fp8:
            problems.append(f"weight {w!r} is {tags[tensors[w][0]][0]}, not F8_E4M3 or F8_E5M2")
        elif len(tensors[w][1]) != 2:
            problems.append(f"weight {w!r} has shape {list(tensors[w][1])}, not 2-D")
        if not isinstance(sc, str) or sc not in tensors:
            problems.append(f"scale {sc!r} of {w!r} is not {there}")
            continue
        sdt, sshape = tensors[sc]
        if sdt not in codes:
            problems.append(f"scale {sc!r} is {tags[sdt][0]}, not F32, F16 or BF16")
        elif good_block and w in tensors and len(tensors[w][1]) == 2:
            sr, scol = _scale_grid(tensors[w][1], scale_block)
            fits = [(sr, scol)] + ([(), (1,)] if sr == scol == 1 else [(sr,)] if scol == 1 else [])
            if tuple(sshape) not in fits:
                problems.append(f"scale {sc!r} has shape {list(sshape)}; weight {w!r} of shape {list(tensors[w][1])} "
                                f"in blocks {tuple(scale_block)} needs [{sr}, {scol}]")
        if select is not None and sc in select:
            problems.append(f"scale {sc!r} is selected, but scales are consumed")
        if into is not None and sc in into:
            problems.append(f"scale {sc!r} is in into, but scales are consumed")
        target = dtype.get(w) if isinstance(dtype, Mapping) else dtype
        if isinstance(dtype, Mapping) and target is None:
            problems.append(f"weight {w!r} has no target in dtype")
        elif target is not None and (not isinstance(target, torch.dtype) or target not in codes):
            problems.append(f"weight {w!r}: {target} is not a supported target ({supported})")
        else:
            out[w] = target
    if problems:
        raise ValueError(f"{where}: scales: " + "; ".join(problems))
    return out


async def _read_shards(client, volume_id: str, where: str, shards, select, into, dtype, scales, scale_block,
                       staging_bytes: int, ctx, fp8=None, scale_suffix: str = "_scale_inv") -> dict:
    """The body of ``read_safetensors_sharded`` over ``shards`` (``[(path, header length, entries)]``; also
    ``read_safetensors`` and ``read_safetensors_slices`` with ``scales=``, and ``read_safetensors`` with ``fp8=``, over
    one shard).  With ``scales``, the scales load first, unconverted, into temporary tensors (one ``_load_runs``: a
    scale may sit in a later wave, or another shard, than its weight), then everything else (a second ``_load_runs``).
    With ``fp8``, the weights it names are quantized in the one ``_load_runs`` (``_Quant``), their a in one temporary
    array, zeroed once and freed on return."""
    import torch

    by_name = {e[0]: (k, 8 + n + e[3], e) for k, (_, n, entries) in enumerate(shards) for e in entries}
    scaled, consumed, quant = {}, set(), {}
    if fp8 is not None:
        problems = []
        there = "in the checkpoint" if len(shards) > 1 else "in the file"
        quant = _fp8_load_plan(there, {name: (e[1], e[2]) for name, (_, _, e) in by_name.items()},
                               {name: at for name, (_, at, _) in by_name.items()}, fp8, scale_block, scale_suffix,
                               dtype, scales, select, staging_bytes, problems)
        rest = {name: t for name, t in dtype.items() if name not in quant} if isinstance(dtype, Mapping) else dtype
        targets = {}
        try:
            targets = cast_targets(where, rest, [(name, e[1], e[2], at, None) for name, (_, at, e) in by_name.items()
                                                 if name not in quant], 0)
        except ValueError as exc:
            problems.append(str(exc))
        if into is not None:  # its mismatches go in the same error (the weights as E4M3, their scales as F32 grids)
            grids = {}
            for w, sc in quant.items():
                try:
                    grids[sc] = list(_scale_grid(by_name[w][2][2], scale_block))
                except (TypeError, ValueError, ZeroDivisionError):  # a bad scale_block, already reported
                    pass
            want = [(name, torch.float8_e4m3fn if name in quant else targets.get(name, e[1]), e[2], 0, 0)
                    for name, (_, _, e) in by_name.items()] + [(sc, torch.float32, g, 0, 0) for sc, g in grids.items()]
            try:
                _check_into(into, want, ctx, stored={name: e[1] for name, (_, _, e) in by_name.items()
                                                     if name in quant or name in targets})
            except ValueError as exc:
                problems.append(str(exc))
        if problems:
            raise ValueError(f"{where}: fp8: " + "; ".join(problems))
    if scales:
        there = "in the checkpoint" if len(shards) > 1 else "in the file"
        scaled = _scale_targets(where, there, dtype, scales, scale_block,
                                {name: (e[1], e[2]) for name, (_, _, e) in by_name.items()}, select, into)
        consumed = set(scales.values())
    plans = []  # (shard, name, stored dtype, result shape, runs)
    if select is None:
        for name, (k, at, (_, dt, shape, lo, hi)) in by_name.items():
            if name not in consumed:
                plans.append((k, name, dt, shape, [(at, hi - lo, hi - lo, 1)] if hi > lo else []))
    else:
        unknown = [name for name in select if name not in by_name]
        if unknown:
            raise ValueError(f"{where}: no tensors named {', '.join(repr(u) for u in unknown)}")
        for name, index in select.items():
            k, at, (_, dt, shape, _, _) = by_name[name]
            bounds, kept = _slice_bounds(name, shape, index)
            result = [hi - b for (b, hi), keep in zip(bounds, kept) if keep]
            plans.append((k, name, dt, result, _slice_runs(shape, bounds, dt.itemsize, at)))
    sliced = select is not None
    rest = dtype
    if scaled and isinstance(dtype, Mapping):
        rest = {name: t for name, t in dtype.items() if name not in scaled}
    if fp8 is None:
        targets = cast_targets(where, rest, [(name, dt, shape, by_name[name][1], None)
                                             for _, name, dt, shape, _ in plans if name not in scaled], 0, sliced=sliced)
    targets.update(scaled)
    targets.update({name: torch.float8_e4m3fn for name in quant})
    grids = {sc: list(_scale_grid(by_name[w][2][2], scale_block)) for w, sc in quant.items()}
    if into is not None:
        if fp8 is None:  # with fp8, checked above
            _check_into(into, [(name, targets.get(name, dt), shape, 0, 0) for _, name, dt, shape, _ in plans], ctx,
                        sliced=sliced, stored={name: dt for _, name, dt, *_ in plans if name in targets})
        tensors = [into[name] for _, name, *_ in plans]
        qscales = {sc: into[sc] for sc in quant.values()}
    else:
        tensors = [DeviceFile._Source._new_tensor(shape, targets.get(name, dt), ctx) for _, name, dt, shape, _ in plans]
        qscales = {sc: DeviceFile._Source._new_tensor(grids[sc], torch.float32, ctx) for sc in quant.values()}
    qs = {}
    if quant:  # every weight's a, in one array zeroed with one memset
        amax = DeviceFile._Source._new_tensor([sum(g[0] * g[1] for g in grids.values())], torch.float32, ctx).zero_()
        at = 0
        for w, sc in quant.items():
            (R, C), (br, bc), n = by_name[w][2][2], scale_block, grids[sc][0] * grids[sc][1]
            qs[w] = _Quant(amax[at : at + n], qscales[sc].view(-1), by_name[w][1], R, C, min(R, br or R),
                           min(C, bc or C), by_name[w][2][1])
            at += n
    dequant = {}
    if scaled:  # the scales of the weights with a byte to load, whole and unconverted, into temporary tensors
        needed = sorted({scales[name] for _, name, _, _, rs in plans if name in scaled and rs},
                        key=lambda sc: (by_name[sc][0], by_name[sc][1]))
        temps = {sc: DeviceFile._Source._new_tensor(by_name[sc][2][2], by_name[sc][2][1], ctx) for sc in needed}
        per = {}  # shard -> [its scale tensors, runs, packed bytes so far]
        for sc in needed:
            k, at, (_, _, _, lo, hi) = by_name[sc]
            ts, runs, base = per.setdefault(k, [[], [], 0])
            if hi > lo:
                runs.append(((at, hi - lo, hi - lo, 1), base, None))
            ts.append(temps[sc])
            per[k][2] = base + hi - lo
        files = []
        for k in sorted(per):
            ts, runs, _ = per[k]
            if runs:
                start = min(F for (F, _, _, _), _, _ in runs)
                end = max(F + W for (F, W, _, _), _, _ in runs)
                files.append((shards[k][0], runs, DeviceFile._over(DeviceFile._Source(ts, BOUNCE_BYTES)), start, end))
        await _load_runs(client, volume_id, files, staging_bytes)
        for w in scaled:
            if scales[w] in temps:
                (R, C), (br, bc) = by_name[w][2][2], scale_block
                dequant[w] = _Dequant(temps[scales[w]], by_name[w][1], R, C, max(1, R if br is None else br),
                                      max(1, C if bc is None else bc))
    per = {}  # shard -> [its result tensors, runs, packed bytes so far]
    for (k, name, dt, _, rs), t in zip(plans, tensors):
        ts, runs, base = per.setdefault(k, [[], [], 0])
        dest = base
        conv = (dt, t.dtype, dequant[name]) if name in dequant else (dt, t.dtype, qs[name]) if name in qs else \
            (dt, t.dtype) if name in targets else None
        for run in rs:
            runs.append((run, dest, conv))
            dest += run[1] * run[3] // dt.itemsize * t.element_size()
        ts.append(t)
        per[k][2] = base + t.numel() * t.element_size()
    files = []
    for k in sorted(per):
        ts, runs, _ = per[k]
        if runs:
            start = min(F for (F, _, _, _), _, _ in runs)
            end = max(F + (R - 1) * P + W for (F, W, P, R), _, _ in runs)
            files.append((shards[k][0], runs, DeviceFile._over(DeviceFile._Source(ts, BOUNCE_BYTES)), start, end))
    await _load_runs(client, volume_id, files, staging_bytes)
    out = {}
    for (_, name, *_), t in zip(plans, tensors):
        out[name] = t
        if name in quant:
            out[quant[name]] = qscales[quant[name]]
    return out


_ZIP_TAIL = 1 << 16  # the end of a torch.save file read first: its end records and, usually, its central directory
_ZIP_TRAILER = 1 << 12  # read before the central directory too: torch.save's version and serialization id records


def _check_format_version(path: str, prefix: str, small: dict) -> None:
    """The archive's format version as torch's own reader checks it (the range this torch reads), ``ValueError``
    otherwise: ``torch._C.PyTorchFileReader`` over a zip of the version records alone."""
    import zipfile

    import torch

    b = BytesIO()
    with zipfile.ZipFile(b, "w") as z:
        for name in ("version", ".data/version"):
            if name in small:
                z.writestr(prefix + name, small[name])
    try:
        torch._C.PyTorchFileReader(BytesIO(b.getvalue()))
    except RuntimeError as exc:
        raise ValueError(f"{path}: {exc}") from None


class _ArchiveRecords:
    """What ``torch.serialization._load`` reads a torch.save archive through (the reader interface of
    ``torch._C.PyTorchFileReader``, record names without the archive prefix): the small records from host memory, and
    for every ``data/<key>`` record the pickle references a new, empty storage of the record's size
    (``DeviceFile._Source._empty``), kept in ``storages`` to be filled afterwards."""

    def __init__(self, small: dict, data: dict, ctx):
        self.small, self.data, self.ctx = small, data, ctx
        self.storages: dict = {}  # record name -> uint8 tensor over the storage

    def has_record(self, name: str) -> bool:
        return name in self.small or name in self.data

    def get_record(self, name: str) -> bytes:
        if name not in self.small:
            raise ValueError(f"torch.save archive: no record {name!r} among its small records")
        return self.small[name]

    def get_all_records(self) -> list[str]:
        return [*self.small, *self.data]

    def serialization_id(self) -> str:
        return self.small.get(".data/serialization_id", b"").decode("ascii", "replace")

    def get_storage_from_record(self, name: str, nbytes: int, _storage_type):
        r = self.data.get(name)
        if r is None:
            raise ValueError(f"torch.save archive: the pickle references {name!r}, which has no record")
        if r.size != nbytes:
            raise ValueError(f"torch.save archive: the pickle gives {name!r} {nbytes} bytes, its record holds {r.size}")
        if name not in self.storages:
            self.storages[name] = DeviceFile._Source._empty(nbytes, self.ctx)
        return self.storages[name]


class _StorageWaves:
    """The ``plan`` of ``read_torch_save``'s waves: the staged span starts at file offset ``span_at``, the storages'
    ``records`` are the segments of the destination file, in file order.  Before a wave's storage bytes are written,
    the local header of every storage whose data starts in it is checked against the central directory; it is in this
    wave's or the previous wave's slots (those are not refilled yet).  Also the ``_Skeleton`` reads over those slots."""

    def __init__(self, path: str, records, span_at: int):
        self.path, self.records, self.span_at = path, records, span_at
        self.seg_at = np.concatenate([[0], np.cumsum([r.size for r in records])]).tolist()
        self.window: list = [[], []]  # (offset in the span, length, buffer offset) of the previous and current slices
        self.checked = self.open = 0  # storages whose header was checked / the first one not completely written
        self.buf = None

    def read(self, off: int, n: int) -> bytes:
        out, lo = bytearray(), off - self.span_at
        for o, m, a in self.window[0] + self.window[1]:
            x, y = max(lo, o), min(lo + n, o + m)
            if x < y:
                out += self.buf[a + x - o : a + y - o].tobytes()
        if len(out) != n:
            raise ValueError(f"{self.path}: bytes [{off}, {off + n}) of a local header are not in the staging buffer")
        return bytes(out)

    def u(self, off: int, n: int) -> int:
        return int.from_bytes(self.read(off, n), "little")

    def __call__(self, wave, at, buf):
        self.buf = buf
        self.window = [self.window[1], [(o, m, a) for (_, o, m), a in zip(wave, at)]]
        lo, hi = wave[0][1] + self.span_at, wave[-1][1] + wave[-1][2] + self.span_at  # file offsets of the wave
        recs = self.records
        while self.checked < len(recs) and recs[self.checked].data < hi:
            r = recs[self.checked]
            got = device_file._local_data_offset(self, r)
            if got != r.data:
                raise ValueError(f"{self.path}: the local header of {r.name!r} puts its data at {got}, but the central "
                                 f"directory leaves room for it only at {r.data} (its data must end right before the "
                                 f"next record)")
            self.checked += 1
        while self.open < len(recs) and recs[self.open].data + recs[self.open].size <= lo:
            self.open += 1
        ranges, offsets = [], []
        for i in range(self.open, len(recs)):
            d, n = recs[i].data, recs[i].size
            if d >= hi:
                break
            for (_, o, m), a in zip(wave, at):
                x, y = max(d, o + self.span_at), min(d + n, o + self.span_at + m)
                if x < y:
                    ranges.append((0, self.seg_at[i] + x - d, y - x))
                    offsets.append(a + x - o - self.span_at)
        return ranges, offsets


def _crc_mismatches(pairs) -> list[str]:
    """``pairs``: (record, computed CRC-32); the records whose stored CRC-32 is not 0 and differs, as text."""
    return [f"{r.name} (stored {r.crc:08x}, computed {c:08x})" for r, c in pairs if r.crc and r.crc != c]


async def read_torch_save(client, volume_id: str, path: str, *, weights_only: bool = True,
                          staging_bytes: int = 256 << 20):
    """The torch.save checkpoint at ``path``, loaded as ``torch.load(f, map_location=f"cuda:{ctx.device}",
    weights_only=weights_only)`` loads the file's bytes (same structure, types, dtypes, shapes, strides and values;
    storages shared in the file are shared in the result, CPU-saved ones are on the device too), without assembling the
    image in host memory or HBM, and with the stored CRC-32 of every record it reads checked (unreferenced data records
    are neither read nor checked).

    The end of the file (end records, central directory, and the small records after the data records: ``version``,
    ``.data/serialization_id``), then the region before the first data record (``data.pkl`` and the other small
    records) come through host memory in ranged reads.  The small records' CRC-32s are checked with zlib, the format
    version as torch's own reader checks it, and ``data.pkl`` is unpickled by torch's own loader (``find_class``
    remapping, the ``weights_only`` allow-lists, the tensor rebuilds), every storage it references being a new, empty
    tensor on the device.  Only then does one ``VolumeGetFile2`` call name the blocks from the first referenced data
    record to the end of the last one: at most five calls in all for an archive torch.save wrote, whatever the number
    of storages.  The blocks go through ``staging_bytes`` of page-locked memory (two halves, as
    ``read_file_into_device``) and every complete wave writes the storages' bytes in it with one ``load_ranges`` call.
    Where each storage's data starts is taken from the central directory before the download (its data ends right
    before the next record's local header, less its data descriptor); each storage's own local header, read from the
    staging buffer, must name the record and put the data there, else ``ValueError`` (an archive with bytes between
    records, for one).  Last, one ``crc32_device`` call on the current stream covers every loaded storage with a stored
    CRC-32 (torch writes 0 when CRCs are off: not checked), and the values are read back once.  A mismatch raises
    ``ExecutionError`` naming every bad record.  On return the bytes are ordered before work enqueued later on the
    current stream.

    ``ValueError`` before any GET of the data region: not a zip archive (the legacy format included), a TorchScript
    archive, a compressed record, a format version this torch does not read, a ``byteorder`` other than little, a
    storage whose data is not 16-byte aligned, a storage whose size differs from its record's (``torch.load`` refuses
    it too) or that has no record; torch's ``pickle.UnpicklingError`` for a global ``weights_only`` refuses;
    ``FileNotFoundError`` for a missing path."""
    import pickle
    import zlib

    import torch

    BS = blob_utils.BLOCK_SIZE
    if staging_bytes < 2 * BS:
        raise ValueError(f"staging_bytes must hold two blocks ({2 * BS} bytes), got {staging_bytes}")
    ctx = blob_utils.get_context()
    size = (await _get_file2(client, volume_id, path, 0, 1)).size
    # the end of the file as ONE piece: a central directory field may lie on either side of any read's edge
    end_at = max(0, size - _ZIP_TAIL)
    end = bytearray(await _read_range_host(client, volume_id, path, end_at, size - end_at))

    async def extend_end(lo: int):
        nonlocal end, end_at
        if lo < end_at:
            end = bytearray(await _read_range_host(client, volume_id, path, lo, end_at - lo)) + end
            end_at = lo

    try:
        _, cd_off = device_file._zip_directory(device_file._Skeleton([(end_at, end)]))
    except ValueError:
        raise ValueError(f"{path} is not a torch.save zip archive (no end-of-central-directory record)") from None
    if not 0 <= cd_off <= size:
        raise ValueError(f"{path}: the central directory offset {cd_off} lies outside the {size}-byte file")
    await extend_end(max(0, cd_off - _ZIP_TRAILER))
    records = sorted(device_file._central_directory(device_file._Skeleton([(end_at, end)])), key=lambda r: r.local)
    if not records:
        raise ValueError(f"{path}: the zip archive holds no records")
    prefix = records[0].name.split("/", 1)[0] + "/"
    if any(not r.name.startswith(prefix) for r in records):
        raise ValueError(f"{path}: the archive's records do not share one prefix ({prefix!r})")
    rel = {r.name[len(prefix) :]: r for r in records}
    if "constants.pkl" in rel:
        raise ValueError(f"{path} is a TorchScript archive; load it with torch.jit.load")
    if "data.pkl" not in rel:
        raise ValueError(f"{path}: the archive has no data.pkl record")
    data = {n: r for n, r in rel.items() if n.startswith("data/")}
    # Where every data record's bytes must start, known before any of them is downloaded: its data ends where the next
    # local header (or the central directory) begins, less the data descriptor torch's zip writer puts after every
    # non-empty record (ZIP64-sized from 4 GiB on).  Each local header is checked against this as it arrives.
    for r, nxt in zip(records, [r.local for r in records[1:]] + [cd_off]):
        desc = 0 if not r.flags & 8 else 24 if r.local >= 0xFFFFFFFF or r.size >= 0xFFFFFFFF else 16
        r.data = nxt - desc - r.size
    head_end = min([r.local for r in data.values()] + [cd_off])
    # the small records after the data records (torch.save: version, .data/serialization_id) end up in the end piece
    await extend_end(min([r.local for n, r in rel.items() if n not in data and r.local > head_end], default=end_at))
    pieces = [(end_at, end)]
    if head_end >= end_at:
        await extend_end(0)
        pieces = [(0, end)]
    elif head_end:
        pieces.insert(0, (0, bytearray(await _read_range_host(client, volume_id, path, 0, head_end))))
    sk = device_file._Skeleton(pieces)
    small = {}
    for n, r in rel.items():
        if n not in data:
            r.data = device_file._local_data_offset(sk, r)
            if r.local < head_end and r.data + r.size > head_end:
                raise ValueError(f"{path}: record {r.name!r} runs into the data records")
            small[n] = sk.read(r.data, r.size)
    bad = _crc_mismatches((rel[n], zlib.crc32(b)) for n, b in small.items())
    if bad:
        raise ExecutionError(f"{path}: CRC-32 mismatch in " + ", ".join(bad))
    _check_format_version(path, prefix, small)
    if small.get("byteorder", b"little") != b"little":
        raise ValueError(f"{path}: byteorder {small['byteorder']!r} is not supported (only little-endian archives)")

    reader = _ArchiveRecords(small, data, ctx)
    loader = torch.serialization._weights_only_unpickler if weights_only else pickle
    obj = torch.serialization._load(reader, lambda storage, _location: storage, loader, encoding="utf-8")

    loads = sorted(((data[n], t) for n, t in reader.storages.items() if t.numel()), key=lambda e: e[0].local)
    for r, _ in loads:
        if r.data % 16:
            raise ValueError(f"{path}: the data of {r.name!r} starts at {r.data}, which is not 16-byte aligned")
    if not loads:
        return obj
    span_at = loads[0][0].local & ~15  # 16-aligned, so that every storage sits 16-aligned in its block slot
    span_end = loads[-1][0].data + loads[-1][0].size
    slices = await _block_slices(client, volume_id, path, span_at, span_end - span_at)
    dst = DeviceFile._over(DeviceFile._Source([t for _, t in loads], BOUNCE_BYTES))
    plan = _StorageWaves(path, [r for r, _ in loads], span_at)
    def load(wave, at, buf, ctx):
        ranges, src_offsets = plan(wave, at, buf)
        return load_ranges([dst], ranges, buf, src_offsets, ctx=ctx)

    await _load_in_waves(slices, load, staging_bytes, None, lambda **_: None)
    checked = [(r, t) for r, t in loads if r.crc]
    if checked:
        crc = DeviceFile._Source._empty(4 * len(checked), ctx).view(torch.int32)
        ctx.crc32_device([t.data_ptr() for _, t in checked], [t.numel() for _, t in checked], crc.data_ptr(),
                         DeviceFile._Source._current_stream(ctx))
        bad = _crc_mismatches(zip([r for r, _ in checked], crc.cpu().numpy().view(np.uint32).tolist()))
        if bad:
            raise ExecutionError(f"{path}: CRC-32 mismatch in " + ", ".join(bad))
    return obj


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

