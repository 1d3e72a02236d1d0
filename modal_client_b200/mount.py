"""Mount creation on the GPU hash path: select files, checksum them, dedupe, upload, register.

Counterpart of the upload half of ``_Mount`` (py/modal/mount.py): entries (``_MountFile`` :111-134, ``_MountDir``
:136-196), ``_select_files`` (:103-108), ``_Mount._get_files`` (:465-485) and ``_Mount._load_mount`` (:487-622).
The RPC sequence per file is the reference's -- ``MountPutFile(sha256_hex)`` existence check, upload as inline
data or through ``blob_upload_file``, poll ``MountPutFile(data|data_blob_id)`` until the server has it, then one
``MountGetOrCreate`` with the file index -- what changes is the two steps around the hash path:

* *checksums*: the reference runs ``get_file_upload_spec_from_path`` per file on a ``ThreadPoolExecutor``
  (:467-481); here all selected files form ONE GPU batch (``blob_utils.get_file_upload_specs``: native reader
  threads -> pinned ring -> fused SHA-256+MD5 kernel).
* *dedupe*: the reference keeps an ``accounted_hashes`` set and tests it file by file on the event loop
  (:498,518-534); here the first occurrence of every content is computed on the GPU over the digest table
  (``b200h_dedupe_host``), before the first RPC goes out.

Out of scope (control plane): ``_Object`` hydration, resolver / load-context plumbing, deployment lookups,
``_MountedPythonModule`` import machinery, the status-row UI.  ``load_mount`` takes the stub and the few fields
``_load_mount`` reads from them.
"""
from __future__ import annotations

import abc
import asyncio
import dataclasses
import os
import time
import typing
import warnings
from collections.abc import Callable, Sequence
from pathlib import Path, PurePosixPath

from . import _wire, blob_utils
from ._lib import B200HashError
from ._logging import logger
from .async_utils import bounded_map
from .blob_utils import FileUploadSpec
from .exception import ExecutionError, MountUploadTimeoutError

ROOT_DIR: PurePosixPath = PurePosixPath("/root")  # mount.py:38
MOUNT_PUT_FILE_CLIENT_TIMEOUT = 10 * 60  # 10 min max for transferring files (mount.py:39)


class _MountEntry(metaclass=abc.ABCMeta):  # mount.py:89-100
    @abc.abstractmethod
    def description(self) -> str: ...

    @abc.abstractmethod
    def get_files_to_upload(self) -> typing.Iterator[tuple[Path, PurePosixPath]]: ...

    @abc.abstractmethod
    def top_level_paths(self) -> list[tuple[Path, PurePosixPath]]: ...


@dataclasses.dataclass
class _MountFile(_MountEntry):
    """One local file at ``remote_path`` (mount.py:111-134)."""

    local_file: Path
    remote_path: PurePosixPath

    def description(self) -> str:
        return str(self.local_file)

    def get_files_to_upload(self):
        local_file = Path(self.local_file).resolve()
        if not local_file.exists():
            raise FileNotFoundError(f"local file {local_file} does not exist")
        yield local_file, PurePosixPath(self.remote_path)

    def top_level_paths(self):
        return [(Path(self.local_file), PurePosixPath(self.remote_path))]


def _ignore_nothing(_path: Path) -> bool:
    return False


@dataclasses.dataclass
class _MountDir(_MountEntry):
    """A local directory below ``remote_path``; ``ignore(relative_path) -> True`` drops a file (mount.py:136-196).
    An ``ignore`` object exposing ``can_prune_directories()`` (the reference's pattern matchers do) also prunes
    whole directories during the walk."""

    local_dir: Path
    remote_path: PurePosixPath
    ignore: Callable[[Path], bool] = _ignore_nothing
    recursive: bool = True

    def description(self) -> str:
        return str(Path(self.local_dir).expanduser().absolute())

    def _walk(self, top_dir: Path, prune: bool):
        for root, dirs, files in os.walk(top_dir, topdown=True):
            if prune:  # in-place edit of dirs: os.walk does not descend into ignored directories
                dirs[:] = [d for d in dirs if not self.ignore(Path(os.path.join(root, d)).relative_to(top_dir))]
            for file in files:
                yield os.path.join(root, file)

    def get_files_to_upload(self):
        # no eager .resolve(): that would "rename" symlinked files (reference comment at mount.py:162-163)
        local_dir = Path(self.local_dir).expanduser().absolute()
        if not local_dir.exists():
            raise FileNotFoundError(f"local dir {local_dir} does not exist")
        if not local_dir.is_dir():
            raise NotADirectoryError(f"local dir {local_dir} is not a directory")
        if self.recursive:
            can_prune = getattr(self.ignore, "can_prune_directories", None)
            gen = self._walk(local_dir, bool(can_prune and can_prune()))
        else:
            gen = (e.path for e in os.scandir(local_dir) if e.is_file())
        for local_filename in gen:
            local_path = Path(local_filename)
            rel = local_path.relative_to(local_dir)
            if not self.ignore(rel):
                yield local_path.resolve(), PurePosixPath(self.remote_path) / rel.as_posix()

    def top_level_paths(self):
        return [(Path(self.local_dir), PurePosixPath(self.remote_path))]


def _select_files(entries: Sequence[_MountEntry]) -> list[tuple[Path, PurePosixPath]]:
    """Union of what the entries select (a set, so overlapping entries do not duplicate a pair) -- mount.py:103-108.
    Sorted here so that the batch, the dedupe and the resulting file index are deterministic."""
    all_files: set[tuple[Path, PurePosixPath]] = set()
    for entry in entries:
        all_files |= set(entry.get_files_to_upload())
    return sorted(all_files, key=lambda lr: (lr[1].as_posix(), str(lr[0])))


def get_file_specs(entries: Sequence[_MountEntry]) -> list[FileUploadSpec]:
    """``_Mount._get_files`` (mount.py:465-485) as one batch.  A file that disappears between selection and
    reading (editors' temp files) is ignored with a log line, like the reference's ``except FileNotFoundError``."""
    selected = []
    for p, r in _select_files(entries):
        if p.is_file():
            selected.append((p, r))
        else:  # removed between selection and now (editors' temp files): the reference's `except FileNotFoundError`
            logger.info(f"Ignoring file not found: {p}")
    logger.debug(f"Computing checksums for {len(selected)} files on the GPU")
    try:
        return blob_utils.get_file_upload_specs([(p, r, None) for p, r in selected])
    except (B200HashError, OSError) as exc:
        # something vanished or became unreadable after the is_file() check: redo file by file so that only the
        # offending files are dropped (still the GPU path; there is no CPU hashing anywhere)
        logger.info(f"batched checksum failed ({exc}); retrying file by file")
        specs = []
        for p, r in selected:
            try:
                specs.append(blob_utils.get_file_upload_spec_from_path(p, r))
            except FileNotFoundError as exc2:
                logger.info(f"Ignoring file not found: {exc2}")
        return specs


def _description(entries: Sequence[_MountEntry]) -> str:
    return ", ".join(e.description() for e in entries)


async def load_mount(
    entries: Sequence[_MountEntry],
    stub,
    *,
    deployment_name: str | None = None,
    namespace: int = 0,
    environment_name: str = "",
    app_id: str | None = None,
    allow_overwrite: bool = False,
    build_start: float | None = None,
    build_validation: str = "error",
    n_concurrent_uploads: int = 64,
):
    """Checksum, dedupe and upload the files of ``entries``, then register the mount: the data path of
    ``_Mount._load_mount`` (mount.py:487-622).  Returns the ``MountGetOrCreate`` response.

    ``build_start`` / ``build_validation`` reproduce the "file modified during build" check (:523-532):
    with a ``build_start`` timestamp, a path whose mtime is newer raises (``"error"``), warns (``"warn"``)
    or is accepted (``"ignore"``)."""
    t0 = time.monotonic()
    message_label = _description(entries)
    specs = await asyncio.to_thread(get_file_specs, entries)
    first, n_distinct = await asyncio.to_thread(blob_utils.first_occurrence_of_specs, specs)
    logger.debug(f"Creating mount {message_label}: {len(specs)} files, {n_distinct} distinct contents")

    blob_upload_concurrency = asyncio.Semaphore(16)  # limit uploads of large files (mount.py:503)
    total_uploads, total_bytes = 0, 0

    async def _put_file(file_spec: FileUploadSpec) -> None:
        nonlocal total_uploads, total_bytes
        # catch local modifications between the start of a build and the upload (mount.py:523-532)
        if build_validation != "ignore" and build_start is not None and file_spec.source_is_path:
            if os.stat(file_spec.source_description).st_mtime > build_start:
                msg = f"{file_spec.source_description} was modified during build process."
                if build_validation == "error":
                    raise ExecutionError(msg)
                warnings.warn(msg)
        response = await stub.MountPutFile(_wire.MountPutFileRequest(sha256_hex=file_spec.sha256_hex))
        if response.exists:
            return
        total_uploads += 1
        total_bytes += file_spec.size
        if file_spec.use_blob:
            logger.debug(f"Creating blob file for {file_spec.source_description} ({file_spec.size} bytes)")
            async with blob_upload_concurrency:
                with file_spec.source() as fp:
                    blob_id = await blob_utils.blob_upload_file(fp, stub, sha256_hex=file_spec.sha256_hex,
                                                                md5_hex=file_spec.md5_hex)
            request2 = _wire.MountPutFileRequest(data_blob_id=blob_id, sha256_hex=file_spec.sha256_hex)
        else:
            content = file_spec.content
            if content is None:
                content = await asyncio.to_thread(file_spec.read_content)
            request2 = _wire.MountPutFileRequest(data=content, sha256_hex=file_spec.sha256_hex)
        start_time = time.monotonic()
        while time.monotonic() - start_time < MOUNT_PUT_FILE_CLIENT_TIMEOUT:
            response = await stub.MountPutFile(request2)
            if response.exists:
                return
        raise MountUploadTimeoutError(f"Mounting of {file_spec.source_description} timed out")

    # only the first occurrence of a content is checked / sent; the others just appear in the index.
    # n_concurrent_uploads in flight, as async_map(..., concurrency=64) does in the reference (mount.py:573-577)
    await bounded_map([s for i, s in enumerate(specs) if first[i] == i], _put_file, concurrency=n_concurrent_uploads)

    files = [_wire.MountFile(filename=s.mount_filename, sha256_hex=s.sha256_hex, mode=s.mode) for s in specs]
    if not files:
        logger.warning(f"Mount of '{message_label}' is empty.")
    if deployment_name:
        creation_type = (_wire.OBJECT_CREATION_TYPE_CREATE_IF_MISSING if allow_overwrite
                         else _wire.OBJECT_CREATION_TYPE_CREATE_FAIL_IF_EXISTS)
        req = _wire.MountGetOrCreateRequest(deployment_name=deployment_name, namespace=namespace,
                                            environment_name=environment_name, object_creation_type=creation_type,
                                            files=files)
    elif app_id is not None:
        req = _wire.MountGetOrCreateRequest(object_creation_type=_wire.OBJECT_CREATION_TYPE_ANONYMOUS_OWNED_BY_APP,
                                            files=files, app_id=app_id)
    else:
        req = _wire.MountGetOrCreateRequest(object_creation_type=_wire.OBJECT_CREATION_TYPE_EPHEMERAL, files=files,
                                            environment_name=environment_name)
    resp = await stub.MountGetOrCreate(req)
    logger.debug(f"Uploaded {total_uploads} new files and {total_bytes} bytes in {time.monotonic() - t0}s")
    return resp


__all__ = ["ROOT_DIR", "MOUNT_PUT_FILE_CLIENT_TIMEOUT", "_MountEntry", "_MountFile", "_MountDir", "_select_files",
           "get_file_specs", "load_mount"]
