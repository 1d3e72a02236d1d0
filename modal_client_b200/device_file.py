"""A read-only file object over bytes that live in GPU memory: one CUDA tensor, or a safetensors image of many.

``DeviceFile(t)`` lets a buffer that lives in GPU memory -- a checkpoint shard, a safetensors image, an embedding
table -- go wherever the upload functions accept a ``BinaryIO``, without first copying the whole buffer to host memory.
``DeviceFile.safetensors(state_dict)`` is the same for a whole checkpoint: a file whose bytes are exactly what
``safetensors.torch.save(state_dict)`` would produce, made of the tensors where they are (plus a small header), so the
image is never assembled, neither in host memory nor in HBM.

* volumefs2 (``VolumeUploadContextManager2.put_file`` / ``FileUploadSpec2.from_fileobj``) recognises it and trims and
  hashes its 8 MiB blocks in place (``hash_parts``) with one ``b200h_hash_segment_parts_device`` call, whatever
  tensors the file is made of; only the blocks that straddle tensor boundaries are gathered.  Only the (trimmed
  length, SHA-256) table comes to the host, and afterwards only the trimmed bytes of the blocks the server reports
  missing are read.
* every other consumer (volumefs1 ``put_file``, ``get_file_upload_spec_from_fileobj``, ``blob_upload_file``) reads it
  like any other stream.  Those digests are one serial chain over the whole object and gain nothing from the GPU.

``read`` / ``readinto`` copy device -> host through one page-locked bounce buffer of bounded size (16 MiB by default),
so host memory never has to hold the tensors.  ``bytes_to_host`` counts what has crossed.  The readers ``reopen()``
hands out share the tensors, the bounce buffer and that counter.  The tensors must not change while an upload reads
them.

``stage_ranges(files, ranges, dst, dst_offsets)`` is the bulk route off the device: any byte ranges of any number of
device files into a page-locked buffer with ONE ``b200h_copy_ranges_to_host`` call, after which the tensors are not
needed for those bytes.  The volumefs2 uploader uses it for the missing blocks when it is given
``device_staging_bytes``.  ``load_ranges(files, ranges, src, src_offsets)`` is the way back: ranges of a page-locked
buffer into the files' tensors with ONE ``b200h_copy_ranges_from_host`` call (``volume.read_file_into_device``), and
``load_boxes(files, boxes, src)`` the strided form: rows of a page-locked buffer, any distance apart and at any phase,
packed into the files with ONE ``b200h_copy_boxes_from_host`` call (``volume.read_safetensors_slices``).
``load_cast_boxes(files, boxes, src)`` is ``load_boxes`` whose elements change type on the way (F32, F16, BF16), with
ONE ``b200h_copy_cast_boxes_from_host`` call (``volume.read_safetensors(..., dtype=...)``).
``load_scaled_boxes(files, boxes, src)`` dequantizes FP8 boxes with their block scales on the way, with ONE
``b200h_copy_scaled_boxes_from_host`` call (``volume.read_safetensors(..., dtype=..., scales=...)``).

``safetensors_shards(state_dict, max_shard_size=...)`` is a checkpoint in the Hugging Face Hub's sharded layout: the
files ``huggingface_hub.save_torch_state_dict`` writes, each shard a ``DeviceFile.safetensors``, plus the index.

``DeviceFile.safetensors(..., fp8=names)`` (and ``safetensors_shards``) exports weights as block-scaled FP8 E4M3 with
their F32 scales: the scales are computed on the device by ONE ``b200h_fp8_block_scales`` call, and the weights are
quantized as the file's bytes leave the device (``b200h_hash_scaled_segment_parts_device``,
``b200h_copy_scaled_ranges``), never held quantized in HBM.
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
    pinned bounce buffer, a lock, a byte counter.

    With ``casts`` -- ``(src_type, dst_type)`` ``_lib.DT_*`` codes per segment, equal (0, 0) for one that converts
    nothing -- the file is the segments' converted images: segment s contributes its elements as ``dst_type``, and
    every offset and count (``seg_start``, ``nbytes``, ``bytes_to_host``) is in image bytes.  The converted bytes are
    made on the way out, by the context ``ctx``, and never held in HBM.

    With ``scales`` as well -- per segment ``(amax_ptr, scale_count, R, C, block_rows, block_cols)``, or None for one
    that does not quantize -- a segment whose ``dst_type`` is ``_lib.DT_F8E4M3`` is its weight quantized with those
    amax values (one image byte per element), and every copy and hash is a scaled call."""

    device_type = "cuda"

    def __init__(self, tensors, bounce_bytes: int, casts=None, ctx=None, scales=None):
        import torch

        self._attach(tensors, bounce_bytes, casts, ctx, scales)
        device = self.segments[0].device
        self.stream = torch.cuda.Stream(device)
        # everything already queued on the caller's stream (the kernels that produced the tensors) runs first
        self.stream.wait_stream(torch.cuda.current_stream(device))
        self.stream_handle = self.stream.cuda_stream

    def _attach(self, tensors, bounce_bytes: int, casts=None, ctx=None, scales=None):
        """``tensors``: one tensor, or a non-empty list of them in file order."""
        import torch

        self.tensors = list(tensors) if isinstance(tensors, (list, tuple)) else [tensors]  # keep the storages alive
        self.segments = [t.reshape(-1).view(torch.uint8) for t in self.tensors]
        self.casts, self.ctx, self.scales = casts, ctx, scales
        size = {_lib.DT_F32: 4, _lib.DT_F16: 2, _lib.DT_BF16: 2, _lib.DT_F8E4M3: 1}
        self.seg_start = [0]  # file offset of every segment, then the size
        for i, s in enumerate(self.segments):
            st, dt = casts[i] if casts else (0, 0)
            self.seg_start.append(self.seg_start[-1] + (s.numel() // size[st] * size[dt] if st != dt else s.numel()))
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

    def _mark(self):
        """-> a callable that blocks until everything queued on this source's stream so far has completed."""
        import torch

        event = torch.cuda.Event()
        event.record(self.stream)
        return event.synchronize

    def _after_current(self):
        """Order this source's stream after everything the current stream holds now."""
        import torch

        self.stream.wait_stream(torch.cuda.current_stream(self.segments[0].device))

    def _publish(self):
        """Make the current stream wait for everything queued on this source's stream so far; -> a callable that blocks
        until that work has completed."""
        import torch

        event = torch.cuda.Event()
        event.record(self.stream)
        torch.cuda.current_stream(self.segments[0].device).wait_event(event)
        return event.synchronize

    @classmethod
    def _new_tensor(cls, shape, dtype, ctx):
        import torch

        return torch.empty(shape, dtype=dtype, device=f"cuda:{ctx.device}")

    @classmethod
    def _to_device(cls, data: bytes, ctx):
        import torch

        return torch.frombuffer(bytearray(data), dtype=torch.uint8).to(f"cuda:{ctx.device}")

    @classmethod
    def _pinned(cls, n: int):
        import torch

        return torch.empty(n, dtype=torch.uint8, pin_memory=True)

    @classmethod
    def _empty(cls, n: int, ctx):
        import torch

        return torch.empty(n, dtype=torch.uint8, device=f"cuda:{ctx.device}")

    @classmethod
    def _current_stream(cls, ctx) -> int:
        """The current stream as the library takes it.  PyTorch's default stream is the legacy NULL stream, but a NULL
        stream means the context's own stream to the library, so it is named cudaStreamLegacy (1) instead."""
        import torch

        return torch.cuda.current_stream(ctx.device).cuda_stream or 1

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
        from several segments; with casts, by one ``copy_cast_ranges`` call)."""
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
                    if self.scales:
                        ptrs, lens, first = _file_table([self])
                        self.ctx.copy_scaled_ranges(ptrs, lens, *_types([self]), _scales([self]), first,
                                                    [(0, pos + done, k)], bounce, [0], self.stream_handle)
                        filled = k
                    elif self.casts:
                        ptrs, lens, first = _file_table([self])
                        self.ctx.copy_cast_ranges(ptrs, lens, *_types([self]), first, [(0, pos + done, k)], bounce, [0],
                                                  self.stream_handle)
                        filled = k
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
    ptrs, lens, first = _file_table(sources)
    n = sum(-(-src.nbytes // part_len) for src in sources)
    with lead._on_stream():
        d_sha, d_md5, d_trim = _outputs(n, flags, lead.segments[0].device)
        if any(src.scales for src in sources):
            got = ctx.hash_scaled_segment_parts_device(ptrs, lens, *_types(sources), _scales(sources), first, part_len,
                                                       flags, _ptr(d_sha), _ptr(d_md5), _ptr(d_trim),
                                                       lead.stream_handle)
        elif any(src.casts for src in sources):
            got = ctx.hash_cast_segment_parts_device(ptrs, lens, *_types(sources), first, part_len, flags, _ptr(d_sha),
                                                     _ptr(d_md5), _ptr(d_trim), lead.stream_handle)
        else:
            got = ctx.hash_segment_parts_device(ptrs, lens, first, part_len, flags, _ptr(d_sha), _ptr(d_md5),
                                                _ptr(d_trim), lead.stream_handle)
        assert got == n
        return _fetch(d_sha, d_md5, d_trim)


def hash_parts_many(files: list["DeviceFile"], part_len: int, flags: int = _lib.SHA256 | _lib.MD5, ctx=None):
    """``DeviceFile.hash_parts`` of several files at once: every file's parts (one or more segments each), file-major,
    digested by ONE ``b200h_hash_segment_parts_device`` call on the first file's stream, which is ordered after every
    file's stream (``b200h_hash_cast_segment_parts_device`` when any of the files converts its tensors).  -> (sha uint8[n,32] | None, md5 uint8[n,16] | None, trimmed uint64[n])."""
    return _hash_sources([f._src for f in files], ctx or get_context(), part_len, flags)


class Staged:
    """Ranges of device files on their way into a page-locked host buffer (``stage_ranges``)."""

    def __init__(self, dst: np.ndarray, spans: list[tuple[int, int]], done):
        self._dst, self._spans, self._done = dst, spans, done

    def wait(self) -> None:
        """Blocks until the copy has completed (call it through ``asyncio.to_thread`` from a coroutine).  From then on
        the files' tensors are not needed for these ranges."""
        if self._done is not None:
            self._done()
            self._done = None

    def view(self, i: int) -> memoryview:
        """The bytes of range ``i`` where they are in the destination buffer (no copy); valid after ``wait()``."""
        at, n = self._spans[i]
        return memoryview(self._dst[at : at + n])


def stage_ranges(files: list["DeviceFile"], ranges, dst: np.ndarray, dst_offsets, ctx=None) -> Staged:
    """Copy ``ranges`` -- ``(index into files, offset, length)`` each -- of device files into ``dst``, a uint8 array
    over page-locked memory from ``ctx.host_alloc``; range i lands at ``dst[dst_offsets[i]:]`` (offsets multiples of
    16, destinations disjoint; the layout is the caller's).  ONE ``b200h_copy_ranges_to_host`` call (one kernel launch)
    whatever the files are made of, enqueued on the first file's stream, which is ordered after every file's stream;
    ONE ``b200h_copy_cast_ranges`` call instead when any of the files converts its tensors, and ONE
    ``b200h_copy_scaled_ranges`` call when any of them quantizes.
    Returns at once; ``wait()`` on the result blocks until the bytes are in ``dst``.  Every file's ``bytes_to_host``
    grows by the bytes of its ranges."""
    ctx = ctx or get_context()
    sources, ranges, offsets = _range_args(files, ranges, dst_offsets, "dst_offsets")
    if not sources:
        return Staged(dst, [], None)
    lead = sources[0]
    ptrs, lens, first = _file_table(sources)
    with lead._on_stream():
        if any(src.scales for src in sources):
            ctx.copy_scaled_ranges(ptrs, lens, *_types(sources), _scales(sources), first, ranges, dst, offsets,
                                   lead.stream_handle)
        elif any(src.casts for src in sources):
            ctx.copy_cast_ranges(ptrs, lens, *_types(sources), first, ranges, dst, offsets, lead.stream_handle)
        else:
            ctx.copy_ranges_to_host(ptrs, lens, first, ranges, dst, offsets, lead.stream_handle)
        done = lead._mark()
    for f, _, n in ranges:
        with sources[f].lock:
            sources[f].bytes_to_host += n
    return Staged(dst, [(at, n) for at, (_, _, n) in zip(offsets, ranges)], done)


def _file_table(sources: list[_TensorBytes]):
    """(segment pointers, lengths, file_first_seg) of ``sources``, with the first one's stream ordered after the
    others'."""
    lead = sources[0]
    ptrs, lens, first = [], [], [0]
    for src in sources:
        lead._after(src)
        ptrs += [s.data_ptr() if s.numel() else 0 for s in src.segments]
        lens += [s.numel() for s in src.segments]
        first.append(len(lens))
    return ptrs, lens, first


def _types(sources: list[_TensorBytes]):
    """(src_types, dst_types) of every segment of ``sources``, in ``_file_table`` order ((0, 0): the bytes as they
    are)."""
    pairs = [pair for src in sources for pair in (src.casts or [(0, 0)] * len(src.segments))]
    return [st for st, _ in pairs], [dt for _, dt in pairs]


def _scales(sources: list[_TensorBytes]):
    """Every segment's ``(amax_ptr, scale_count, R, C, block_rows, block_cols)`` of ``sources``, in ``_file_table``
    order (zeros for a segment that does not quantize)."""
    return [q or (0,) * 6 for src in sources for q in (src.scales or [None] * len(src.segments))]


def _range_args(files: list["DeviceFile"], ranges, offsets, offsets_name: str):
    """(sources, ranges as int triples, offsets as ints) of a ``stage_ranges`` / ``load_ranges`` call, checked."""
    sources = [f._src for f in files]
    ranges = [(int(f), int(o), int(n)) for f, o, n in ranges]
    offsets = [int(o) for o in offsets]
    if len(offsets) != len(ranges):
        raise ValueError(f"{offsets_name} needs one entry per range")
    if ranges and not sources:
        raise ValueError("ranges without files")
    return sources, ranges, offsets


class Loaded:
    """Ranges of a page-locked host buffer on their way into device files (``load_ranges``)."""

    def __init__(self, done):
        self._done = done

    def wait(self) -> None:
        """Blocks until the copy has completed (call it through ``asyncio.to_thread`` from a coroutine).  Only from
        then on may the host change the source buffer."""
        if self._done is not None:
            self._done()
            self._done = None


def load_ranges(files: list["DeviceFile"], ranges, src: np.ndarray, src_offsets, ctx=None) -> Loaded:
    """Write ``src[src_offsets[i]:]`` -- ``src`` a uint8 array over page-locked memory from ``ctx.host_alloc``, offsets
    multiples of 16 -- into range i = ``(index into files, offset, length)`` of device files; no device byte may belong
    to two ranges.  The mirror of ``stage_ranges``: ONE ``b200h_copy_ranges_from_host`` call (one kernel launch),
    enqueued on the first file's stream, which is ordered after every file's stream and after the current stream (the
    tensors may have been read since the files were made; they are not overwritten before that work).  The current
    stream then waits for the copy, so work enqueued on it later sees the bytes without a host synchronisation.
    Returns at once; ``wait()`` on the result blocks until the kernel has read ``src``.  ``DeviceFile`` itself stays a
    read-only file object: this is the one way bytes get into its tensors."""
    ctx = ctx or get_context()
    sources, ranges, offsets = _range_args(files, ranges, src_offsets, "src_offsets")
    if not sources:
        return Loaded(None)
    lead = sources[0]
    lead._after_current()
    ptrs, lens, first = _file_table(sources)
    with lead._on_stream():
        ctx.copy_ranges_from_host(ptrs, lens, first, ranges, src, offsets, lead.stream_handle)
    return Loaded(lead._publish())  # outside the block: the caller's current stream is the one that waits


def load_boxes(files: list["DeviceFile"], boxes, src: np.ndarray, ctx=None) -> Loaded:
    """Write boxes of ``src`` -- a uint8 array over page-locked memory from ``ctx.host_alloc`` -- into device files:
    box i = ``(index into files, offset, width, rows, src_offset, src_pitch)`` writes ``rows`` rows of ``width`` bytes,
    row r from ``src[src_offset + r * src_pitch:]`` (no alignment needed; ``src_pitch >= width`` when ``rows > 1``),
    packed into bytes ``[offset, offset + rows * width)`` of its file; no device byte may belong to two boxes.  ONE
    ``b200h_copy_boxes_from_host`` call (one kernel launch, none when every box is empty), ordered as ``load_ranges``:
    on the first file's stream, after every file's stream and the current stream, and the current stream then waits
    for the copy.  Returns at once; ``wait()`` on the result blocks until the kernel has read ``src``."""
    ctx = ctx or get_context()
    sources = [f._src for f in files]
    boxes = [tuple(int(x) for x in b) for b in boxes]
    if any(len(b) != 6 for b in boxes):
        raise ValueError("a box is (file, offset, width, rows, src_offset, src_pitch)")
    return _load_boxes(ctx, "copy_boxes_from_host", sources, boxes, src)


def _load_boxes(ctx, entry: str, sources: list[_TensorBytes], boxes, src: np.ndarray, *extra) -> Loaded:
    """The body of ``load_boxes`` and ``load_cast_boxes``: ONE call of ``ctx``'s ``entry`` with the checked boxes (and
    ``extra`` after them), on the first file's stream, ordered as ``load_ranges``."""
    if boxes and not sources:
        raise ValueError("boxes without files")
    if not sources:
        return Loaded(None)
    lead = sources[0]
    lead._after_current()
    ptrs, lens, first = _file_table(sources)
    with lead._on_stream():
        getattr(ctx, entry)(ptrs, lens, first, boxes, *extra, src, lead.stream_handle)
    return Loaded(lead._publish())


def cast_dtypes() -> dict:
    """The torch dtypes ``load_cast_boxes`` converts between, with their ``_lib.DT_*`` codes."""
    import torch

    return {torch.float32: _lib.DT_F32, torch.float16: _lib.DT_F16, torch.bfloat16: _lib.DT_BF16}


def cast_targets(path: str, dtype, entries, data_start: int, sliced: bool = False) -> dict:
    """{name: target dtype} of the tensors of ``entries`` -- ``(name, dtype, shape, data offset, end)`` each, as
    ``volume._safetensors_entries`` gives them (the selected ones for ``read_safetensors_slices``; a state dict's tensors
    for ``DeviceFile.safetensors``) -- that ``dtype`` converts: ``None``; one of float32, float16 and bfloat16 for every
    F32 / F16 / BF16 tensor of another dtype, integer and bool tensors unchanged; or ``{name: such a dtype}``.  Every
    problem in one ``ValueError``: another floating dtype under a single dtype, a mapped name that is not there, an
    unsupported target or source, and a tensor to convert whose file offset (``data_start`` + its data offset) is not a
    multiple of its element size."""
    if dtype is None:
        return {}
    import torch

    codes, tags = cast_dtypes(), _st_dtypes()
    by_name = {e[0]: e for e in entries}
    problems, want = [], {}
    supported = "float32, float16 or bfloat16"
    if isinstance(dtype, Mapping):
        for name, target in dtype.items():
            if name not in by_name:
                problems.append(f"{name!r} is in dtype but not {'selected' if sliced else 'in the file'}")
            else:
                want[name] = target
    elif not isinstance(dtype, torch.dtype) or dtype not in codes:
        problems.append(f"{dtype} is not a supported target ({supported})")
    else:
        for name, src, *_ in entries:
            if src in codes:
                want[name] = dtype
            elif tags[src][0][0] in "FC":  # F64, F8_*, F4, C64: floating, but not converted
                problems.append(f"{name!r} is {tags[src][0]}, which does not convert to {dtype}")
    out = {}
    for name, target in want.items():
        _, src, _, lo, _ = by_name[name]
        if not isinstance(target, torch.dtype) or target not in codes:
            problems.append(f"{name!r}: {target} is not a supported target ({supported})")
        elif src not in codes:
            problems.append(f"{name!r} is {tags[src][0]}; only F32, F16 and BF16 tensors convert")
        elif src != target:
            if (data_start + lo) % src.itemsize:
                problems.append(f"{name!r} starts at file offset {data_start + lo}, not a multiple of its element size "
                                f"{src.itemsize}")
            out[name] = target
    if problems:
        raise ValueError(f"{path}: dtype: " + "; ".join(problems))
    return out


def _fp8_plan(tensors: Mapping, dtype, fp8, scale_block, scale_suffix, problems: list) -> dict:
    """{weight: scale name} of the names in ``fp8``, in the order of ``tensors``, for ``DeviceFile.safetensors(...,
    fp8=...)``; every problem is appended to ``problems``: unknown or repeated names, weights that are not 2-D, empty or
    F32 / F16 / BF16, a bad ``scale_block`` or ``scale_suffix``, a scale name that is already a name, a name that
    ``dtype`` maps too, and a weight that shares its storage with another name."""
    import torch

    if isinstance(fp8, str):
        fp8 = None  # a single name is a common slip: refused, not read as its characters
    try:
        names = list(fp8)
    except TypeError:
        problems.append("fp8 must be an iterable of tensor names")
        return {}
    if not (isinstance(scale_block, (tuple, list)) and len(scale_block) == 2 and
            all(b is None or (isinstance(b, int) and not isinstance(b, bool) and b >= 1) for b in scale_block)):
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
            problems.append(f"{n!r} is in fp8 but not in the tensors")
        else:
            want.add(n)
    owners: dict = {}  # storage -> names
    for n, t in tensors.items():
        if isinstance(t, torch.Tensor) and t.untyped_storage().nbytes():
            owners.setdefault((t.device, t.untyped_storage().data_ptr()), []).append(n)
    plan = {}
    for n, t in tensors.items():
        if n not in want:
            continue
        if not isinstance(t, torch.Tensor) or t.dim() != 2 or t.numel() == 0:
            problems.append(f"{n!r} is not a non-empty 2-D tensor; fp8 quantizes 2-D weights")
        elif t.dtype not in codes:
            problems.append(f"{n!r} is {t.dtype}; only float32, float16 and bfloat16 weights quantize")
        else:
            others = [o for o in owners.get((t.device, t.untyped_storage().data_ptr()), []) if o != n]
            if others:
                problems.append(f"{n!r} shares its storage with {', '.join(map(repr, others))}; a quantized weight "
                                f"must have a storage of its own")
        if isinstance(dtype, Mapping) and n in dtype:
            problems.append(f"{n!r} is in both fp8 and dtype")
        if scale_suffix is not None:
            if n + scale_suffix in tensors:
                problems.append(f"the scale of {n!r}, {n + scale_suffix!r}, is already a tensor name")
            plan[n] = n + scale_suffix
    return plan


def _fp8_targets(label: str, tensors: Mapping, dtype, plan: dict, problems: list) -> dict:
    """``cast_targets`` of the tensors that do not quantize (a ``dtype`` mapping without the quantized names); its
    problems go to ``problems``."""
    if dtype is None:
        return {}
    rest = {k: v for k, v in dtype.items() if k not in plan} if isinstance(dtype, Mapping) else dtype
    try:
        return cast_targets(label, rest, [(n, t.dtype, t.shape, 0, None) for n, t in tensors.items() if n not in plan],
                            0)
    except ValueError as exc:
        problems.append(str(exc))
        return {}


def load_cast_boxes(files: list["DeviceFile"], boxes, src: np.ndarray, ctx=None) -> Loaded:
    """``load_boxes`` with a conversion: box i = ``(index into files, offset, width, rows, src_offset, src_pitch,
    src_dtype, dst_dtype)``, two different torch dtypes of ``cast_dtypes()``, converts the ``rows * width / itemsize``
    elements of type ``src_dtype`` (``width`` and ``src_pitch`` count source bytes) to ``dst_dtype`` -- rounding to
    nearest even exactly as torch's CUDA ``.to()`` does -- and writes them packed from byte ``offset`` of its file.
    Every row must start at a multiple of the source itemsize in ``src``'s memory, and a box's destination must lie in
    one tensor of its file at a multiple of the destination itemsize.  ONE ``b200h_copy_cast_boxes_from_host`` call,
    ordered exactly as ``load_boxes``."""
    ctx = ctx or get_context()
    sources = [f._src for f in files]
    if any(len(b) != 8 for b in boxes):
        raise ValueError("a box is (file, offset, width, rows, src_offset, src_pitch, src_dtype, dst_dtype)")
    codes = cast_dtypes()
    for b in boxes:
        for dt in b[6:]:
            if dt not in codes:
                raise ValueError(f"load_cast_boxes converts between {', '.join(map(str, codes))}, not {dt}")
    boxes = [tuple(int(x) for x in b[:6]) + (codes[b[6]], codes[b[7]]) for b in boxes]
    return _load_boxes(ctx, "copy_cast_boxes_from_host", sources, boxes, src)


def fp8_dtypes() -> dict:
    """The FP8 torch dtypes ``load_scaled_boxes`` dequantizes, with their ``_lib.DT_*`` codes."""
    import torch

    return {torch.float8_e4m3fn: _lib.DT_F8E4M3, torch.float8_e5m2: _lib.DT_F8E5M2}


def load_scaled_boxes(files: list["DeviceFile"], boxes, src: np.ndarray, ctx=None) -> Loaded:
    """``load_cast_boxes`` for FP8 weights with block scales: box i = ``(index into files, offset, width, rows,
    src_offset, src_pitch, src_dtype, dst_dtype, scales, first_elem, R, C, block_rows, block_cols)``.  ``src_dtype`` is
    ``torch.float8_e4m3fn`` or ``torch.float8_e5m2`` (one byte per element, so ``width`` and ``src_pitch`` count both),
    ``dst_dtype`` one of ``cast_dtypes()``, and ``scales`` a contiguous float32 / float16 / bfloat16 tensor on the
    context's device holding ``ceil(R / block_rows) * ceil(C / block_cols)`` scales or more, row-major.  Element c of row
    r of the box is element ``first_elem + r * src_pitch + c`` of an R x C weight W; it lands as
    ``(W.float() * S_expanded).to(dst_dtype)``, bit for bit torch's result on CUDA (a block of R or more rows, C or more
    columns, is the whole dimension).  The scales must not change until the copy has completed.  ONE
    ``b200h_copy_scaled_boxes_from_host`` call, ordered exactly as ``load_boxes``."""
    import torch

    ctx = ctx or get_context()
    sources = [f._src for f in files]
    if any(len(b) != 14 for b in boxes):
        raise ValueError("a box is (file, offset, width, rows, src_offset, src_pitch, src_dtype, dst_dtype, scales, "
                         "first_elem, R, C, block_rows, block_cols)")
    codes, fp8 = cast_dtypes(), fp8_dtypes()
    out = []
    for b in boxes:
        if b[6] not in fp8:
            raise ValueError(f"load_scaled_boxes dequantizes {', '.join(map(str, fp8))}, not {b[6]}")
        if b[7] not in codes:
            raise ValueError(f"load_scaled_boxes converts to {', '.join(map(str, codes))}, not {b[7]}")
        s = b[8]
        if not isinstance(s, torch.Tensor) or s.dtype not in codes or not s.is_contiguous():
            raise ValueError("a box's scales are a contiguous float32, float16 or bfloat16 tensor on the context's "
                             "device")
        out.append(tuple(int(x) for x in b[:6]) + (fp8[b[6]], codes[b[7]], s.data_ptr(), codes[s.dtype], s.numel())
                   + tuple(int(x) for x in b[9:]))
    return _load_boxes(ctx, "copy_scaled_boxes_from_host", sources, out, src)


def _f32_device(t, what: str):
    import torch

    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or not t.is_contiguous():
        raise ValueError(f"{what} is a contiguous float32 tensor on the context's device")
    return t.data_ptr()


def _quant_boxes(boxes) -> list:
    """The ``_lib`` form of ``load_fp8_amax_boxes`` / ``load_quant_boxes`` boxes, checked."""
    codes = cast_dtypes()
    if any(len(b) != 13 for b in boxes):
        raise ValueError("a box is (file, offset, width, rows, src_offset, src_pitch, src_dtype, amax, first_elem, R, "
                         "C, block_rows, block_cols)")
    out = []
    for b in boxes:
        if b[6] not in codes:
            raise ValueError(f"quantizing boxes take {', '.join(map(str, codes))}, not {b[6]}")
        ptr = _f32_device(b[7], "a box's amax")
        out.append(tuple(int(x) for x in b[:6]) + (codes[b[6]], _lib.DT_F8E4M3, ptr, b[7].numel())
                   + tuple(int(x) for x in b[8:]))
    return out


def load_fp8_amax_boxes(files: list["DeviceFile"], boxes, src: np.ndarray, ctx=None) -> Loaded:
    """The first half of quantizing F32 / F16 / BF16 weights to FP8 E4M3 as they arrive in ``src`` (a uint8 array over
    page-locked memory from ``ctx.host_alloc``): box i = ``(index into files, offset, width, rows, src_offset,
    src_pitch, src_dtype, amax, first_elem, R, C, block_rows, block_cols)``, ``src_dtype`` one of ``cast_dtypes()``
    (``width`` and ``src_pitch`` count source bytes).  The element at source byte c of row r of the box is element
    ``first_elem + (r * src_pitch + c) / itemsize`` of an R x C weight; the bits of its |x| widened to F32 are
    max-reduced into its block's value of ``amax`` (a contiguous float32 tensor on the context's device of
    ``ceil(R / block_rows) * ceil(C / block_cols)`` values or more, row-major, zeros before a weight's first box).  The
    box's destination in its file (one byte per element) is checked as ``load_quant_boxes`` checks it, and not written.
    ONE ``b200h_fp8_amax_boxes_from_host`` call, ordered exactly as ``load_boxes``."""
    ctx = ctx or get_context()
    return _load_boxes(ctx, "fp8_amax_boxes_from_host", [f._src for f in files], _quant_boxes(boxes), src)


def load_quant_boxes(files: list["DeviceFile"], boxes, bands, src: np.ndarray, ctx=None) -> Loaded:
    """The second half: band i = ``(amax, scales, first, count)`` finalizes blocks ``[first, first + count)`` of a
    weight (``amax`` and ``scales`` contiguous float32 tensors on the context's device: a clamped in place, s = a *
    RN(1 / 448)), then every element of the boxes (as for ``load_fp8_amax_boxes``, whose every block is finalized by now)
    is quantized as the FP8 export quantizes it, q = E4M3(RN(x * RN(RN(1 / a) * 448))), and written packed, one byte
    per element, from byte ``offset`` of its file, into one tensor at any address.  ONE
    ``b200h_copy_quant_boxes_from_host`` call, ordered exactly as ``load_boxes``."""
    ctx = ctx or get_context()
    out = []
    for b in bands:
        if len(b) != 4:
            raise ValueError("a band is (amax, scales, first, count)")
        a, s = _f32_device(b[0], "a band's amax"), _f32_device(b[1], "a band's scales")
        if not 0 <= int(b[2]) <= int(b[2]) + int(b[3]) <= min(b[0].numel(), b[1].numel()):
            raise ValueError(f"band ({int(b[2])}, {int(b[3])}) reaches past its amax or scales")
        out.append((a + 4 * int(b[2]), s + 4 * int(b[2]), int(b[3])))
    return _load_boxes(ctx, "copy_quant_boxes_from_host", [f._src for f in files], _quant_boxes(boxes), src, out)


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


# -------------------------------------------------------------------------------------------- torch.save
#
# A torch.save file is a zip archive of stored (uncompressed) records: data.pkl, a few small ones, one ``data/<key>``
# record per storage holding the whole untyped storage, ``version`` and last ``.data/serialization_id``, then the
# central directory.  ``torch.save`` under ``torch.serialization.skip_data()`` writes all of it except the storage
# bytes, which it skips with ``seek(n, SEEK_CUR)``; in that skeleton the CRC-32 of every data record is 0, and so is
# its contribution to the last 20 digits of the serialization id.  DeviceFile.torch_save keeps the skeleton's pieces
# on the host, takes the storages where they are, has their CRC-32s computed on the device and writes them (and the
# id they determine) into the skeleton.

_ZIP_LOCAL, _ZIP_CENTRAL, _ZIP_DESCRIPTOR = 0x04034B50, 0x02014B50, 0x08074B50
_ZIP_END, _ZIP64_END, _ZIP64_LOCATOR = 0x06054B50, 0x06064B50, 0x07064B50
_ID_RECORD = ".data/serialization_id"
_MASK64 = (1 << 64) - 1


class _SkeletonWriter:
    """The ``f`` torch.save writes into under ``skip_data()``: keeps its writes as pieces and the skipped spans as
    gaps (where the storages go), never a checkpoint-sized buffer."""

    def __init__(self):
        self.pieces: list[tuple[int, bytearray]] = []  # (file offset, bytes), in file order
        self.gaps: list[tuple[int, int]] = []  # (file offset, length) of every skipped span
        self.pos = 0

    def write(self, b) -> int:
        b = memoryview(b).cast("B")
        if self.pieces and self.pieces[-1][0] + len(self.pieces[-1][1]) == self.pos:
            self.pieces[-1][1].extend(b)
        else:
            self.pieces.append((self.pos, bytearray(b)))
        self.pos += len(b)
        return len(b)

    def seek(self, offset: int, whence: int = os.SEEK_SET) -> int:
        if whence != os.SEEK_CUR or offset < 0:
            raise ValueError("torch.save skeleton: only forward relative seeks are expected")
        if offset:
            self.gaps.append((self.pos, offset))
        self.pos += offset
        return self.pos

    def tell(self) -> int:
        return self.pos

    def flush(self):
        pass


class _Skeleton:
    """Read / patch the skeleton's bytes by file offset (every field lies inside one piece)."""

    def __init__(self, pieces):
        self.pieces = pieces
        self.starts = [o for o, _ in pieces]

    def _at(self, off: int, n: int):
        k = bisect.bisect_right(self.starts, off) - 1
        if k < 0 or off + n > self.starts[k] + len(self.pieces[k][1]):
            raise ValueError(f"torch.save layout: bytes [{off}, {off + n}) are not in the skeleton")
        return self.pieces[k][1], off - self.starts[k]

    def read(self, off: int, n: int) -> bytes:
        buf, at = self._at(off, n)
        return bytes(buf[at : at + n])

    def u(self, off: int, n: int) -> int:
        return int.from_bytes(self.read(off, n), "little")

    def patch(self, off: int, data: bytes):
        buf, at = self._at(off, len(data))
        buf[at : at + len(data)] = data


class _ZipRecord:
    __slots__ = ("name", "flags", "crc", "size", "local", "data", "crc_at", "cd_at")


def _zip_directory(sk: _Skeleton) -> tuple[int, int]:
    """(record count, central directory offset) of the archive, from its end-of-central-directory record (in the last
    piece) or the ZIP64 end record it points to."""
    tail_start, tail = sk.pieces[-1][0], sk.pieces[-1][1]
    end = bytes(tail).rfind(_ZIP_END.to_bytes(4, "little"))
    if end < 0:
        raise ValueError("torch.save layout: no end-of-central-directory record")
    end += tail_start
    count, cd_off = sk.u(end + 10, 2), sk.u(end + 16, 4)
    if count == 0xFFFF or cd_off == 0xFFFFFFFF:
        loc = end - 20
        if sk.u(loc, 4) != _ZIP64_LOCATOR:
            raise ValueError("torch.save layout: ZIP64 locator missing")
        z64 = sk.u(loc + 8, 8)
        if sk.u(z64, 4) != _ZIP64_END:
            raise ValueError("torch.save layout: ZIP64 end record missing")
        count, cd_off = sk.u(z64 + 32, 8), sk.u(z64 + 48, 8)
    return count, cd_off


def _central_directory(sk: _Skeleton) -> list[_ZipRecord]:
    """The records of the archive in central-directory order (name, flags, CRC, size, local header offset, and
    ``cd_at``, the offset of the entry), ZIP64 fields included; raises ``ValueError`` on a record that is not stored
    uncompressed."""
    count, at = _zip_directory(sk)
    records = []
    for _ in range(count):
        if sk.u(at, 4) != _ZIP_CENTRAL:
            raise ValueError(f"torch.save layout: no central directory entry at {at}")
        r = _ZipRecord()
        r.cd_at = at
        r.flags, method, r.crc = sk.u(at + 8, 2), sk.u(at + 10, 2), sk.u(at + 16, 4)
        comp, r.size, nlen, xlen, clen = (sk.u(at + 20, 4), sk.u(at + 24, 4), sk.u(at + 28, 2), sk.u(at + 30, 2),
                                          sk.u(at + 32, 2))
        r.local = sk.u(at + 42, 4)
        r.name = sk.read(at + 46, nlen).decode("utf-8")
        x, x_end = at + 46 + nlen, at + 46 + nlen + xlen
        while x < x_end:  # the ZIP64 extra field holds the 32-bit fields that overflowed, in this order
            tag, n = sk.u(x, 2), sk.u(x + 2, 2)
            if tag == 1:
                y = x + 4
                for field in ("size", "comp", "local"):
                    v = {"size": r.size, "comp": comp, "local": r.local}[field]
                    if v == 0xFFFFFFFF:
                        v, y = sk.u(y, 8), y + 8
                        if field == "comp":
                            comp = v
                        else:
                            setattr(r, field, v)
            x += 4 + n
        if method != 0 or comp != r.size:
            raise ValueError(f"torch.save layout: record {r.name!r} is not stored uncompressed")
        records.append(r)
        at = x_end + clen
    return records


def _local_data_offset(sk, r: _ZipRecord) -> int:
    """File offset of ``r``'s data, from its local header (signature, the name as in the central directory, then the
    name and extra lengths).  ``sk``: anything with the ``_Skeleton`` reads that holds the header's bytes."""
    if sk.u(r.local, 4) != _ZIP_LOCAL:
        raise ValueError(f"torch.save layout: no local header for {r.name!r}")
    nlen, xlen = sk.u(r.local + 26, 2), sk.u(r.local + 28, 2)
    if sk.read(r.local + 30, nlen) != r.name.encode("utf-8"):
        raise ValueError(f"torch.save layout: the local header of {r.name!r} names another record")
    return r.local + 30 + nlen + xlen


def _parse_zip(sk: _Skeleton, size: int) -> list[_ZipRecord]:
    """The records of the archive in file order, from its central directory (ZIP64 records included); raises
    ``ValueError`` on anything torch.save does not write (compression, extra bytes between records, ...)."""
    records = _central_directory(sk)
    for r in records:
        r.data = _local_data_offset(sk, r)
        if r.flags & 8:  # CRC and sizes follow the data in a descriptor; the local header's CRC stays 0
            r.crc_at = [r.data + r.size + 4, r.cd_at + 16]
            if sk.u(r.data + r.size, 4) != _ZIP_DESCRIPTOR or sk.u(r.data + r.size + 4, 4) != r.crc:
                raise ValueError(f"torch.save layout: bad data descriptor for {r.name!r}")
        else:
            r.crc_at = [r.local + 14, r.cd_at + 16]
            if sk.u(r.local + 14, 4) != r.crc:
                raise ValueError(f"torch.save layout: local and central CRC of {r.name!r} differ")
    if [r.local for r in records] != sorted(r.local for r in records) or (records and records[-1].data > size):
        raise ValueError("torch.save layout: records out of order")
    return records


def _id_combine(records) -> int:
    """The value behind the last 20 digits of the serialization id: c10::hash_combine over the CRC-32 of every
    non-empty record written before it (torch's writer leaves empty records out)."""
    s = 0
    for r in (r for r in records if r.size):
        s = (s ^ ((r.crc + 0x9E3779B9 + (s << 6) + (s >> 2)) & _MASK64)) & _MASK64
    return s


class _StorageKeys:
    """A pickle module whose Pickler records, for every storage key torch.save's ``persistent_id`` hands out, the
    storage it stands for -- so the data records are matched to their storages by torch's own traversal.  Subclassed by
    torch's PyTorchPickler; pickles exactly as ``pickle.Pickler`` does."""

    __name__ = "torch_save_keys"  # torch.save reads the pickle module's name

    def __init__(self):
        import pickle

        import torch

        keys = self.keys = {}

        class Pickler(pickle.Pickler):
            def __init__(self, *args, **kwargs):
                torch_pid = self.persistent_id  # torch's method: wrapped before the C pickler looks it up

                def persistent_id(obj):
                    if isinstance(obj, torch.Tensor) and obj.device.type == "meta":  # skip_data would drop its storage
                        raise ValueError("DeviceFile.torch_save: a tensor lives on meta, which holds no bytes to save")
                    got = torch_pid(obj)
                    if got is not None and got[0] == "storage":
                        keys.setdefault(got[2], getattr(obj, "_untyped_storage", obj))
                    return got

                self.persistent_id = persistent_id
                super().__init__(*args, **kwargs)

        self.Pickler = Pickler


def torch_save_layout(obj):
    """(skeleton pieces [(offset, bytearray)], [(offset, untyped storage)] in file order, size, parsed records, whether
    CRCs are computed) of ``torch.save(obj)``: the archive without its storage bytes, checked against what the code
    that fills them in assumes."""
    import torch
    from torch.utils.serialization import config

    w, keys = _SkeletonWriter(), _StorageKeys()
    with torch.serialization.skip_data():
        torch.save(obj, w, pickle_module=keys)
    size = w.pos
    if not w.pieces or w.pieces[-1][0] + len(w.pieces[-1][1]) != size:
        raise ValueError("torch.save layout: the archive does not end in written bytes")
    sk = _Skeleton(w.pieces)
    records = _parse_zip(sk, size)
    prefix = records[0].name.split("/", 1)[0] + "/" if records else ""
    data = [r for r in records if r.name.startswith(prefix + "data/")]
    if [r.name for r in data] != [f"{prefix}data/{k}" for k in keys.keys]:
        raise ValueError("torch.save layout: data records do not follow the storage keys")
    gaps = dict(w.gaps)
    storages = []
    for r, (key, st) in zip(data, keys.keys.items()):
        if r.size != st.nbytes() or (r.size and gaps.pop(r.data, None) != r.size):
            raise ValueError(f"torch.save layout: record {r.name!r} does not span its storage's bytes")
        storages.append((r.data, st))
    if gaps:
        raise ValueError("torch.save layout: skipped bytes outside the data records")
    compute_crc = bool(config.save.compute_crc32)
    if records:
        rid = records[-1]
        if rid.name != prefix + _ID_RECORD or rid.size != 40 or not sk.read(rid.data, 40).isdigit():
            raise ValueError("torch.save layout: the last record is not a 40-digit serialization id")
        if compute_crc and (any(r.crc for r in data if r.size) or
                            _id_combine(records[:-1]) != int(sk.read(rid.data + 20, 20))):
            raise ValueError("torch.save layout: the serialization id does not combine the records' CRC-32s")
    return sk, storages, size, records, compute_crc


# ------------------------------------------------------------------------------- sharded safetensors
#
# The Hugging Face Hub's sharded layout, as ``huggingface_hub.save_torch_state_dict`` writes it: names that share a
# storage are reduced to one (``_hub_duplicates``), the rest split greedily in key order on storage sizes
# (``_hub_split``), every shard a safetensors file with ``{"format": "pt"}`` metadata, and with more than one shard a
# ``<pattern>.index.json`` that maps every name to its shard.  The rules are restated here (the library is not a
# dependency); tests/test_safetensors_shards_cpu.py compares the files with the library's.

_SIZE_UNITS = {"TB": 10**12, "GB": 10**9, "MB": 10**6, "KB": 10**3}


def parse_size_to_int(size) -> int:
    """``"5GB"`` -> 5 * 10**9 (units TB, GB, MB, KB, decimal, any case, a fractional value allowed), an int as it is:
    what the Hub takes as ``max_shard_size``."""
    if not isinstance(size, str):
        return size
    text = size.strip()
    unit = text[-2:].upper()
    if unit not in _SIZE_UNITS:
        raise ValueError(f"Unit '{unit}' not supported. Supported units are TB, GB, MB, KB. Got '{text}'.")
    try:
        value = float(text[:-2].strip())
    except ValueError as exc:
        raise ValueError(f"Could not parse the size value from '{text}': {exc}") from None
    return int(value * _SIZE_UNITS[unit])


def _hub_duplicates(tensors: Mapping, discard) -> tuple[dict, list]:
    """({kept name: [removed names]}, [names of every storage no name covers]) of ``tensors``: names whose bytes
    overlap in one storage form a group, and of the names that cover the whole storage the first by name that is not in
    ``discard`` is kept (the first by name when all are).  Every tensor is contiguous."""
    groups: dict = {}
    for name, t in tensors.items():
        st = t.untyped_storage()
        if st.data_ptr() and st.nbytes():
            groups.setdefault((t.device, st.data_ptr(), st.nbytes()), set()).add(name)
    shared = []
    for names in sorted(groups.values()):  # sets sort by inclusion, as the Hub sorts them
        areas = sorted((tensors[n].data_ptr(), tensors[n].data_ptr() + tensors[n].nbytes, n) for n in names)
        _, last_stop, first = areas[0]
        shared.append({first})
        for lo, hi, n in areas[1:]:
            if lo >= last_stop:
                shared.append({n})
            else:
                shared[-1].add(n)
            last_stop = hi
    remove, uncovered = {}, []
    discard = set(discard or ())
    for names in shared:
        complete = {n for n in names if tensors[n].data_ptr() == tensors[n].untyped_storage().data_ptr() and
                    tensors[n].nbytes == tensors[n].untyped_storage().nbytes()}
        if not complete:
            uncovered.append(sorted(names))
            continue
        keep = sorted(complete - discard or complete)[0]
        for n in sorted(names):
            if n != keep:
                remove.setdefault(keep, []).append(n)
    return remove, uncovered


def _hub_split(sizes: Mapping, ids: Mapping, pattern: str, max_size: int) -> tuple[dict, int]:
    """({file name: [tensor names]} in shard order, total size) of the greedy split: in key order, a name whose storage
    id was seen joins that storage's shard at no cost; a storage larger than ``max_size`` is a shard of its own; else
    the current shard is closed when the storage would tip it over ``max_size``."""
    by_id, shards, current, used, total = {}, [], [], 0, 0
    for name, size in sizes.items():
        if ids[name] in by_id:
            by_id[ids[name]].append(name)
            continue
        by_id[ids[name]] = [name]
        total += size
        if size > max_size:
            shards.append([name])
            continue
        if used + size > max_size:
            shards.append(current)
            current, used = [], 0
        current.append(name)
        used += size
    if current:
        shards.append(current)
    for names in by_id.values():
        for shard in shards:
            if names[0] in shard:
                shard += names[1:]
                break
    if len(shards) == 1:
        return {pattern.format(suffix=""): list(sizes)}, total
    return {pattern.format(suffix=f"-{i + 1:05d}-of-{len(shards):05d}"): shard for i, shard in enumerate(shards)}, total


class SafetensorsShards:
    """The files of a sharded safetensors checkpoint (``DeviceFile.safetensors_shards``): ``files``, {file name:
    DeviceFile} in shard order, and ``index``, (file name, bytes) of the index, or None for a single file."""

    def __init__(self, files: dict, index):
        self.files, self.index = files, index

    def put(self, batch, remote_dir) -> None:
        """Queue every shard and the index under ``remote_dir`` on a volumefs2 ``VolumeUploadContextManager2``: the
        batch hashes the blocks of every shard in its one device call, and stages them as it stages any DeviceFile."""
        from pathlib import PurePosixPath

        for name, f in self.files.items():
            batch.put_file(f, PurePosixPath(remote_dir) / name)
        if self.index is not None:
            batch.put_file(io.BytesIO(self.index[1]), PurePosixPath(remote_dir) / self.index[0])


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
    def safetensors(cls, tensors: Mapping, metadata: Mapping | None = None, *, dtype=None, fp8=None,
                    scale_block=(128, 128), scale_suffix: str = "_scale_inv", ctx=None,
                    bounce_bytes: int = BOUNCE_BYTES) -> "DeviceFile":
        """A file whose bytes are the safetensors image of ``tensors`` (``safetensors.torch.save(tensors, metadata)``),
        made of the tensors where they are: the header is built on the host and copied to the device once, every tensor
        is one segment of the file.  Tensors must be contiguous, on the context's device, of a dtype safetensors stores;
        zero-size, 0-d and storage-sharing tensors are fine.  The metadata entries keep the mapping's order (the
        library writes them in no fixed order when there are several).

        ``dtype`` exports the tensors in another dtype, as ``volume.read_safetensors(dtype=...)`` reads them: one of
        torch.float32, float16 and bfloat16 for every F32 / F16 / BF16 tensor (integer and bool tensors unchanged), or
        ``{name: dtype}``.  The file is then exactly ``safetensors.torch.save({k: v.to(target)}, metadata)``, header
        dtypes and data order included, but no converted copy is made: the elements are converted on the device as
        the file's blocks are hashed, staged or read (``b200h_hash_cast_segment_parts_device``,
        ``b200h_copy_cast_ranges``), so HBM holds only the tensors, the header and the digest tables.  A tensor
        already in its target dtype is taken as it is.  Every problem (another floating dtype under a single
        ``dtype``, names not in ``tensors``, unsupported sources or targets) is reported in one ``ValueError`` before
        anything is copied to the device.

        ``fp8`` (an iterable of names of 2-D float32 / float16 / bfloat16 weights) exports those weights as FP8 E4M3
        with block scales, the layout DeepSeek-V3 and the Qwen3 FP8 checkpoints use and ``volume.read_safetensors(...,
        scales=volume.fp8_scales(names, scale_suffix))`` loads: every weight ``w`` is stored as ``F8_E4M3`` and gets an
        F32 tensor ``w + scale_suffix`` of shape ``[ceil(R / rows), ceil(C / columns)]`` for ``scale_block = (rows,
        columns)``, ``None`` meaning the whole dimension (``(1, None)``: per channel; ``(None, None)``: per tensor).
        Element x of block b becomes ``E4M3(x * (448 / a_b))`` and the scale ``a_b / 448``, with ``a_b`` the block's
        amax clamped to at least 1e-4: bit for bit what the widely copied ``per_block_cast_to_fp8`` computes in torch on
        CUDA.  The file is exactly ``safetensors.torch.save(ref, metadata)``, where ``ref`` is ``tensors`` with every
        quantized weight replaced and its scale inserted right after it, and the other tensors converted by ``dtype``
        as above.  The scales are computed on the device at construction (ONE ``b200h_fp8_block_scales`` call on the
        current stream, which does not wait for the GPU) into scale tensors that are segments of the file, plus one F32
        value per block kept for the quantization; no quantized copy of a weight is made: the weights are quantized as
        the file's blocks are hashed, staged or read (``b200h_hash_scaled_segment_parts_device``,
        ``b200h_copy_scaled_ranges``).  The weights must not change while the file is read.  Every problem (see
        ``_fp8_plan``) comes in one ``ValueError`` before anything is copied to the device."""
        if fp8 is not None:
            safetensors_layout(tensors, metadata)  # the names, metadata and dtypes, checked before the rest
            problems = []
            plan = _fp8_plan(tensors, dtype, fp8, scale_block, scale_suffix, problems)
            targets = _fp8_targets("DeviceFile.safetensors", tensors, dtype, plan, problems)
            if problems:
                raise ValueError("DeviceFile.safetensors: " + "; ".join(problems))
            if plan:
                for name, t in tensors.items():
                    ctx = cls._Source._check_tensor(t, ctx, f"DeviceFile.safetensors[{name!r}]")
                ctx = ctx or get_context()
                quant, amax = cls._fp8_scales(tensors, plan, scale_block, ctx)
                plain = {plan[n] if n in plan else n: quant[n][0] if n in plan else t for n, t in tensors.items()}
                return cls._safetensors_scaled(plain, {w: (tensors[w], quant[w][1]) for w in plan}, metadata, targets,
                                               amax, ctx, bounce_bytes)
        if dtype is not None:
            safetensors_layout(tensors, metadata)  # the names, metadata and dtypes, checked before the targets
            targets = cast_targets("DeviceFile.safetensors", dtype,
                                   [(name, t.dtype, t.shape, 0, None) for name, t in tensors.items()], 0)
            if targets:
                return cls._safetensors_cast(tensors, metadata, targets, ctx, bounce_bytes)
        header, ordered = safetensors_layout(tensors, metadata)
        for name, t in ordered:
            ctx = cls._Source._check_tensor(t, ctx, f"DeviceFile.safetensors[{name!r}]")
        head = cls._Source._to_device(header, ctx or get_context())
        return cls._over(cls._Source([head] + [t for _, t in ordered], bounce_bytes))

    @classmethod
    def _safetensors_cast(cls, tensors: Mapping, metadata, targets: dict, ctx, bounce_bytes: int) -> "DeviceFile":
        """``safetensors`` with ``{name: target dtype}`` for the tensors that convert: the layout is that of ``meta``
        stand-ins in the targets, and each converting tensor is a segment of the file that converts."""
        import torch

        for name, t in tensors.items():
            ctx = cls._Source._check_tensor(t, ctx, f"DeviceFile.safetensors[{name!r}]")
        ctx = ctx or get_context()
        stand_ins = {name: torch.empty(t.shape, dtype=targets[name], device="meta") if name in targets else t
                     for name, t in tensors.items()}
        header, ordered = safetensors_layout(stand_ins, metadata)
        codes = cast_dtypes()
        segments, casts = [cls._Source._to_device(header, ctx)], [(0, 0)]
        for name, _ in ordered:
            t = tensors[name]
            segments.append(t)
            casts.append((codes[t.dtype], codes[targets[name]]) if name in targets else (0, 0))
        return cls._over(cls._Source(segments, bounce_bytes, casts, ctx))

    @classmethod
    def _fp8_scales(cls, tensors: Mapping, plan: dict, scale_block, ctx):
        """({weight: (scale tensor, (amax_ptr, scale_count, R, C, block_rows, block_cols))}, the amax buffer) of the
        weights of ``plan``: ONE ``fp8_block_scales`` call on the current stream.  Every scale tensor has a storage of
        its own; the amax values of every weight lie back to back in one buffer, so the call makes one memset."""
        import torch

        codes, jobs, out, at = cast_dtypes(), [], {}, 0
        grids = {w: tuple(1 if b is None else -(-d // b) for d, b in zip(tensors[w].shape, scale_block)) for w in plan}
        amax = cls._Source._new_tensor((sum(g[0] * g[1] for g in grids.values()),), torch.float32, ctx)
        for w in plan:
            t, (g0, g1) = tensors[w], grids[w]
            (R, C), n = t.shape, g0 * g1
            br, bc = (R if scale_block[0] is None else scale_block[0]), (C if scale_block[1] is None else scale_block[1])
            s, a = cls._Source._new_tensor((g0, g1), torch.float32, ctx), amax[at : at + n]
            jobs.append((t.data_ptr(), codes[t.dtype], R, C, br, bc, s.data_ptr(), a.data_ptr()))
            out[w] = (s, (a.data_ptr(), n, R, C, br, bc))
            at += n
        ctx.fp8_block_scales(jobs, cls._Source._current_stream(ctx))
        return out, amax

    @classmethod
    def _safetensors_scaled(cls, plain: Mapping, quant: Mapping, metadata, targets: dict, amax, ctx,
                            bounce_bytes: int = BOUNCE_BYTES) -> "DeviceFile":
        """The file of ``plain`` (tensors stored as they are, or converted to ``targets``; scale tensors among them)
        and ``quant`` ({weight: (tensor, its scales as ``_TensorBytes`` takes them)}, stored as F8_E4M3): the layout is
        that of ``meta`` stand-ins, and each quantized weight is a segment of the file that quantizes."""
        import torch

        stand_ins = {name: torch.empty(t.shape, dtype=targets[name], device="meta") if name in targets else t
                     for name, t in plain.items()}
        stand_ins.update({w: torch.empty(t.shape, dtype=torch.float8_e4m3fn, device="meta") for w, (t, _) in
                          quant.items()})
        header, ordered = safetensors_layout(stand_ins, metadata)
        codes = cast_dtypes()
        segments, casts, scales = [cls._Source._to_device(header, ctx)], [(0, 0)], [None]
        for name, _ in ordered:
            if name in quant:
                t, q = quant[name]
                segments.append(t)
                casts.append((codes[t.dtype], _lib.DT_F8E4M3))
                scales.append(q)
                continue
            t = plain[name]
            segments.append(t)
            casts.append((codes[t.dtype], codes[targets[name]]) if name in targets else (0, 0))
            scales.append(None)
        src = cls._Source(segments, bounce_bytes, casts, ctx, scales)
        src.keep = amax
        return cls._over(src)

    @classmethod
    def safetensors_shards(cls, state_dict: Mapping, *, filename_pattern: str = "model{suffix}.safetensors",
                           max_shard_size="5GB", metadata: Mapping | None = None, dtype=None, fp8=None,
                           scale_block=(128, 128), scale_suffix: str = "_scale_inv",
                           shared_tensors_to_discard=None, ctx=None) -> SafetensorsShards:
        """A checkpoint in the Hugging Face Hub's sharded layout, made of the tensors where they are: every file's
        bytes are exactly what ``huggingface_hub.save_torch_state_dict(state_dict, d, filename_pattern=...,
        max_shard_size=..., metadata=..., shared_tensors_to_discard=...)`` writes into ``d``.

        * Of names that share a storage only one is written, the first by name of those covering the storage that is
          not in ``shared_tensors_to_discard``; every removed name is recorded in the metadata as ``{removed: kept}``
          unless ``metadata`` has that key already.
        * The rest are split in key order: a shard is closed before a storage that would take it over
          ``max_shard_size`` (an int, or ``"5GB"``, ``"512MB"``, ...; decimal units), and a storage larger than that is a
          shard of its own.  One shard is ``filename_pattern.format(suffix="")``; n > 1 are named with the suffix
          ``-0000k-of-0000n`` and come with ``filename_pattern.format(suffix="") + ".index.json"``, ``{"metadata":
          {"total_size": ..., **metadata}, "weight_map": {name: file}}`` as ``json.dump(..., indent=2)`` writes it.
        * Every file is a ``DeviceFile.safetensors`` with metadata ``{"format": "pt"}``, plus ``metadata`` when there
          is a single file (the library writes several entries in no fixed order).

        ``dtype`` is ``DeviceFile.safetensors``'s: the files are then the Hub's of the converted checkpoint -- every
        storage converted once, so tensors that share one still do, as in ``model.to(dtype).state_dict()`` -- split
        on the converted sizes, and every shard converts its elements on the device as it is read, never making a
        converted copy.  Names that share a storage must convert to one dtype.

        ``fp8``, ``scale_block`` and ``scale_suffix`` are ``DeviceFile.safetensors``'s: the files are then the Hub's of
        the quantized checkpoint (every scale right after its weight in key order, split on the quantized sizes, so a
        scale may land in another shard than its weight), with the scales of the whole state dict computed by ONE
        ``b200h_fp8_block_scales`` call before the split.

        Every problem is reported in one ``ValueError`` before anything is copied to the device: a pattern without
        ``{suffix}``, a bad ``max_shard_size``, non-contiguous tensors (the Hub copies them; this call makes no copies
        in HBM), storages that no name covers (the Hub refuses them too), and whatever ``DeviceFile.safetensors``
        refuses."""
        if not isinstance(state_dict, Mapping):
            raise ValueError(f"expected a mapping of str -> torch.Tensor, got {type(state_dict).__name__}")
        problems, valid = [], {}
        try:
            if "{suffix}" not in filename_pattern:
                raise ValueError
            filename_pattern.format(suffix="")
        except (ValueError, KeyError, IndexError, TypeError):
            problems.append(f"filename_pattern {filename_pattern!r} needs exactly one field, {{suffix}}")
        try:
            max_size = parse_size_to_int(max_shard_size)
        except ValueError as exc:
            problems.append(f"max_shard_size: {exc}")
        try:
            safetensors_layout({}, metadata)
        except ValueError as exc:
            problems.append(str(exc))
        for name, t in state_dict.items():
            try:
                safetensors_layout({name: t})
                ctx = cls._Source._check_tensor(t, ctx, f"safetensors_shards[{name!r}]")
                valid[name] = t
            except ValueError as exc:
                problems.append(str(exc))
        targets, plan = {}, {}
        if fp8 is not None and len(valid) == len(state_dict):
            plan = _fp8_plan(state_dict, dtype, fp8, scale_block, scale_suffix, problems)
            targets = _fp8_targets("safetensors_shards", state_dict, dtype, plan, problems)
        elif dtype is not None and len(valid) == len(state_dict):
            try:
                targets = cast_targets("safetensors_shards", dtype,
                                       [(name, t.dtype, t.shape, 0, None) for name, t in state_dict.items()], 0)
            except ValueError as exc:
                problems.append(str(exc))
        remove, uncovered = _hub_duplicates(valid, shared_tensors_to_discard)
        for names in uncovered:
            problems.append(f"no name covers the whole storage of {', '.join(map(repr, names))}")
        for keep, gone in remove.items():
            if len({targets.get(n, valid[n].dtype) for n in [keep] + gone}) > 1:
                problems.append(f"{', '.join(map(repr, [keep] + gone))} share a storage but convert to different "
                                f"dtypes")
        if problems:
            raise ValueError("safetensors_shards: " + "; ".join(problems))
        ctx = ctx or get_context()
        meta = dict(metadata or {})
        for keep, gone in remove.items():
            for n in gone:
                meta.setdefault(n, keep)
        removed = {n for gone in remove.values() for n in gone}
        kept = {n: t for n, t in state_dict.items() if n not in removed}
        quant, amax = cls._fp8_scales(kept, plan, scale_block, ctx) if plan else ({}, None)
        if plan:  # every scale right after its weight: the key order the split follows
            kept = {k: v for n, t in kept.items() for k, v in ([(n, t), (plan[n], quant[n][0])] if n in plan else
                                                                [(n, t)])}
        sizes = {n: t.numel() if n in quant else
                 t.untyped_storage().nbytes() // t.element_size() * targets[n].itemsize if n in targets else
                 t.untyped_storage().nbytes() for n, t in kept.items()}
        ids = {n: (t.device, t.untyped_storage().data_ptr(), sizes[n]) for n, t in kept.items()}
        split, total = _hub_split(sizes, ids, filename_pattern, max_size)
        file_meta = {"format": "pt", **meta} if len(split) == 1 else {"format": "pt"}
        files = {}
        for fname, names in split.items():
            conv = {n: targets[n] for n in names if n in targets}
            if plan:
                files[fname] = cls._safetensors_scaled(
                    {n: kept[n] for n in names if n not in quant}, {n: (kept[n], quant[n][1]) for n in names if n in quant},
                    file_meta, conv, amax, ctx)
            else:
                files[fname] = cls.safetensors({n: kept[n] for n in names}, file_meta, dtype=conv or None, ctx=ctx)
        index = None
        if len(split) > 1:
            body = {"metadata": {"total_size": total, **meta},
                    "weight_map": {n: fname for fname, names in split.items() for n in names}}
            index = (filename_pattern.format(suffix="") + ".index.json", json.dumps(body, indent=2).encode())
        return SafetensorsShards(files, index)

    @classmethod
    def torch_save(cls, obj, *, ctx=None, bounce_bytes: int = BOUNCE_BYTES) -> "DeviceFile":
        """A file whose bytes are exactly ``torch.save(obj, io.BytesIO()).getvalue()`` (records named ``archive/...``),
        made of the storages where they are.  ``obj`` is anything torch.save takes: a state dict, a training
        checkpoint ``{"model": ..., "optim": opt.state_dict(), "step": n}``, nested containers.

        The archive's skeleton (``torch.save`` under ``torch.serialization.skip_data()``: pickle, headers, central
        directory) is built on the host.  Every storage is one segment over its whole untyped storage, in place when it
        is on the context's CUDA device; CPU storages (optimizer ``step`` tensors) are staged to the device together
        with the skeleton's pieces, in one buffer.  Storages on another device raise ``ValueError``.  The CRC-32 of
        every storage is computed on the device (one ``b200h_crc32_device`` call, ordered after the current stream) and
        written into the skeleton with the serialization id it determines; the id record's own CRC-32 comes from the
        device too.  Construction therefore synchronises the current stream twice to read the CRC values back, and not
        at all when ``torch.utils.serialization.config.save.compute_crc32`` is False (the skeleton is then the file) or
        nothing holds a storage.  Only CRC values cross to the host.  The legacy (non-zip) format is not produced."""
        import torch

        ctx = ctx or get_context()
        dev = getattr(ctx, "device", None)
        sk, storages, size, records, compute_crc = torch_save_layout(obj)
        here, staged = [], []  # (file offset, untyped storage) in place / to stage
        for off, st in storages:
            where = st.device
            if where.type == cls._Source.device_type and (where.index == dev or dev in (None, -1)):
                here.append((off, st))
            elif where.type == "cpu":
                staged.append((off, st))
            else:
                raise ValueError(f"DeviceFile.torch_save: a storage lives on {where}, but the file is built on "
                                 f"{cls._Source.device_type}:{dev}")
        as_u8 = lambda st: torch.empty(0, dtype=torch.uint8, device=st.device).set_(st)  # noqa: E731
        # one device buffer: the skeleton's pieces, then the staged storages (16-byte aligned); its host twin is pinned
        layout, at = [], 0
        for off, piece in sk.pieces:
            layout.append((off, at, len(piece)))
            at += len(piece)
        skel_bytes = at
        for off, st in staged:
            at = (at + 15) & ~15
            layout.append((off, at, st.nbytes()))
            at += st.nbytes()
        host, buf = cls._Source._pinned(max(at, 1)), cls._Source._empty(max(at, 1), ctx)
        seg_of = {off: buf[a : a + n] for off, a, n in layout}
        for (off, a, n), (_, st) in zip(layout[len(sk.pieces) :], staged):
            host[a : a + n].copy_(torch.empty(0, dtype=torch.uint8).set_(st))
        if staged:
            buf[skel_bytes:at].copy_(host[skel_bytes:at], non_blocking=True)
        for off, st in here:
            seg_of[off] = as_u8(st)
        hv = host.numpy()
        data = sorted(storages, key=lambda x: x[0])
        if compute_crc and data:
            stream = cls._Source._current_stream(ctx)
            rec_at = {r.data: r for r in records}
            crc = cls._Source._empty(4 * len(data), ctx).view(torch.int32)
            ctx.crc32_device([seg_of[off].data_ptr() if seg_of[off].numel() else 0 for off, _ in data],
                             [seg_of[off].numel() for off, _ in data], crc.data_ptr(), stream)
            for (off, _), c in zip(data, crc.cpu().numpy().view(np.uint32).tolist()):  # synchronisation 1
                rec_at[off].crc = c
                for field in rec_at[off].crc_at:
                    sk.patch(field, c.to_bytes(4, "little"))
            rid = records[-1]
            digits = sk.read(rid.data, 20) + b"%020d" % _id_combine(records[:-1])
            sk.patch(rid.data, digits)
            k = bisect.bisect_right(sk.starts, rid.data) - 1
            a = layout[k][1] + rid.data - sk.starts[k]  # where the id's digits sit in the device buffer
            hv[a : a + 40] = np.frombuffer(digits, np.uint8)
            buf[a : a + 40].copy_(host[a : a + 40], non_blocking=True)
            ctx.crc32_device([buf[a:].data_ptr()], [40], crc.data_ptr(), stream)
            rid.crc = int(crc[:1].cpu().numpy().view(np.uint32)[0])  # synchronisation 2
            for field in rid.crc_at:
                sk.patch(field, rid.crc.to_bytes(4, "little"))
        for (off, piece), (_, a, n) in zip(sk.pieces, layout):
            hv[a : a + n] = np.frombuffer(piece, np.uint8)
        buf[:skel_bytes].copy_(host[:skel_bytes], non_blocking=True)
        segments = [seg_of[off] for off in sorted(seg_of)]
        src = cls._Source(segments, bounce_bytes)
        src.keep = (buf, host)
        assert src.nbytes == size
        return cls._over(src)

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
        """Split the bytes into ceil(size / part_len) parts and digest them where they are, with one
        ``b200h_hash_segment_parts_device`` call whatever tensors the file is made of.
        -> (sha uint8[n,32] | None, md5 uint8[n,16] | None, trimmed uint64[n]); nothing but this table leaves the
        device."""
        return _hash_sources([self._src], ctx or get_context(), part_len, flags)

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


safetensors_shards = DeviceFile.safetensors_shards

__all__ = ["DeviceFile", "BOUNCE_BYTES", "Loaded", "SafetensorsShards", "Staged", "hash_parts_many", "load_boxes",
           "load_cast_boxes", "load_fp8_amax_boxes", "load_quant_boxes", "load_scaled_boxes", "load_ranges", "parse_size_to_int", "safetensors_layout", "safetensors_shards",
           "stage_ranges"]
