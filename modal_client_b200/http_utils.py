"""One shared aiohttp session for object-store PUT/POST, as the reference keeps
(py/modal/_utils/http_utils.py:35-51).  Networking itself is out of scope for the GPU hash path; this exists
so the upload functions that consume the GPU digests have the same shape as the reference's."""
from __future__ import annotations

import asyncio


class ClientSessionRegistry:
    _session = None
    _loop = None

    @classmethod
    def get_session(cls):
        import aiohttp

        loop = asyncio.get_running_loop()
        if cls._session is None or cls._session.closed or cls._loop is not loop:
            cls._session = aiohttp.ClientSession(timeout=aiohttp.ClientTimeout(total=None, sock_connect=30))
            cls._loop = loop
        return cls._session

    @classmethod
    async def close_session(cls):
        if cls._session is not None and not cls._session.closed:
            await cls._session.close()
        cls._session = None
