"""An in-process volumefs2 server that files can be uploaded to and read back from, following the reference's fakes:
``VolumeGetFile2`` names one GET URL per block of the requested byte range, sliced as ``slice_block`` does
(py/test/conftest.py:2913-2966), and the block GET serves the stored (trimmed) block zero-padded to its slice's length,
with the ``error-404`` / ``error-500`` / ``error-503`` tokens (:3415-3445).  Files get there through
``VolumeUploadContextManager2`` (the stub is the content-addressed ``FakeVolumeStub``)."""
from __future__ import annotations

import contextlib
import types

from aiohttp import web

from modal_client_b200 import blob_utils
from tests.blob_server import running_blob_server
from tests.test_device_file_cpu import _ContentAddressedStub
from tests.test_volume_upload import _add_block_route


class NotFoundError(Exception):
    pass


class ReadableVolumeStub(_ContentAddressedStub):
    def __init__(self, host, store, block_size):
        super().__init__(host, store, block_size)
        self.block_hashes: dict[str, list[bytes]] = {}  # path -> the digest of every block, as uploaded
        self.token_version: dict[str, str] = {}  # path -> the version field of its GET tokens ("v2" by default)
        self.get_file_calls: list = []

    async def VolumePutFiles2(self, req):
        out = await super().VolumePutFiles2(req)
        if not out.missing_blocks:
            for f in req.files:
                self.block_hashes[f.path] = [b.contents_sha256 for b in f.blocks]
        return out

    async def VolumeGetFile2(self, req):
        self.get_file_calls.append(req)
        if req.path not in self.block_hashes:
            raise NotFoundError("File not found")
        hashes, BS = self.block_hashes[req.path], self.block_size
        file_size = len(self.volume_files[req.path][0])
        total_start, total_end = req.start, req.start + (req.len or file_size)
        block_start = min(total_start // BS, len(hashes))
        block_end = min(-(total_end // -BS), len(hashes))

        def slice_block(idx):
            lo = total_start % BS if idx == 0 else 0
            hi = (((total_end - 1) % BS) + 1 if total_end > 0 else 0) if idx == block_end - block_start - 1 else BS
            return lo, hi

        version = self.token_version.get(req.path, "v2")
        urls = []
        for idx, digest in enumerate(hashes[block_start:block_end]):
            lo, hi = slice_block(idx)
            urls.append(f"{self.host}/block/test-get-request:{version}:{digest.hex()}:{lo}:{hi - lo}")
        return types.SimpleNamespace(get_urls=urls, size=file_size, start=total_start, len=total_end - total_start)


@contextlib.asynccontextmanager
async def running_volume_server(block_size: int):
    """-> (stub, faults): block PUT and GET routes on one port.  ``faults["statuses"]``: statuses the next GETs answer
    with, one each, before serving normally; ``faults["short"]``: every GET body loses its last byte."""
    faults = {"statuses": [], "short": False, "gets": 0}
    holder = {}
    async with running_blob_server() as (host, store):
        stub = ReadableVolumeStub(host, store, block_size)
        stub.block_puts = 0
        holder["stub"] = stub

        async def get_block(request):
            faults["gets"] += 1
            magic, version, *rest = request.match_info["token"].split(":")
            if magic != "test-get-request":
                return web.Response(status=400, text="bad token")
            if faults["statuses"]:
                status = faults["statuses"].pop(0)
                return web.Response(status=status, text=f"simulated {status}")
            if version.startswith("error-"):
                status = int(version[len("error-"):])
                return web.Response(status=status, text=f"simulated {status}")
            block_id, lo, length = rest
            body = stub.blocks[block_id][int(lo) : int(lo) + int(length)].ljust(int(length), b"\0")
            return web.Response(body=body[:-1] if faults["short"] and body else body)

        app = web.Application(client_max_size=1 << 26)
        app.add_routes([web.put("/block/{token}", _add_block_route(store, holder, block_size)),
                        web.get("/block/{token}", get_block)])
        runner = web.AppRunner(app)
        await runner.setup()
        site = web.TCPSite(runner, "127.0.0.1", 0)
        await site.start()
        stub.host = f"http://127.0.0.1:{site._server.sockets[0].getsockname()[1]}"
        try:
            yield stub, faults
        finally:
            await runner.cleanup()
            await blob_utils.ClientSessionRegistry.close_session()
