"""Request messages of the blob path.  With the real SDK installed these are the generated protobuf
classes (modal_proto/api.proto:811-817); standalone, structurally identical dataclasses stand in so the
upload functions can be driven by any stub object (tests use an in-process fake of BlobCreate)."""
from __future__ import annotations

import dataclasses

try:  # pragma: no cover - only with the real SDK present
    from modal_proto.api_pb2 import BlobCreateRequest, BlobGetRequest  # type: ignore
except Exception:

    @dataclasses.dataclass(slots=True)  # created once per map input: 10^5..10^6 per map
    class BlobCreateRequest:  # type: ignore[no-redef]
        content_md5: str = ""
        content_sha256_base64: str = ""
        content_length: int = 0

    @dataclasses.dataclass
    class BlobGetRequest:  # type: ignore[no-redef]
        blob_id: str = ""


# enum values from modal_proto/api.proto:110-116,164-170
DATA_FORMAT_PICKLE = 1
DATA_FORMAT_CBOR = 4
FUNCTION_CALL_INVOCATION_TYPE_ASYNC = 3
FUNCTION_CALL_INVOCATION_TYPE_SYNC = 4

try:  # pragma: no cover
    from modal_proto.api_pb2 import FunctionInput, FunctionPutInputsItem, FunctionPutInputsRequest  # type: ignore
except Exception:

    @dataclasses.dataclass(slots=True)  # created once per map input: 10^5..10^6 per map
    class FunctionInput:  # type: ignore[no-redef]  (api.proto:2156-2165)
        args: bytes | None = None
        args_blob_id: str | None = None
        data_format: int = DATA_FORMAT_PICKLE
        method_name: str | None = None
        final_input: bool = False

    @dataclasses.dataclass(slots=True)  # created once per map input: 10^5..10^6 per map
    class FunctionPutInputsItem:  # type: ignore[no-redef]  (api.proto:2231-2237)
        idx: int = 0
        input: FunctionInput | None = None
        r2_failed: bool = False
        r2_throughput_bytes_s: int = 0

    @dataclasses.dataclass
    class FunctionPutInputsRequest:  # type: ignore[no-redef]
        function_id: str = ""
        inputs: list = dataclasses.field(default_factory=list)
        function_call_id: str = ""


try:  # pragma: no cover
    from modal_proto.api_pb2 import MapStartOrContinueItem  # type: ignore
except Exception:

    @dataclasses.dataclass(slots=True)  # created once per map input: 10^5..10^6 per map
    class MapStartOrContinueItem:  # type: ignore[no-redef]  (api.proto:2543-2546)
        input: FunctionPutInputsItem | None = None
        attempt_token: str | None = None


# enum ObjectCreationType, modal_proto/api.proto:207-214
OBJECT_CREATION_TYPE_UNSPECIFIED = 0
OBJECT_CREATION_TYPE_CREATE_IF_MISSING = 1
OBJECT_CREATION_TYPE_CREATE_FAIL_IF_EXISTS = 2
OBJECT_CREATION_TYPE_ANONYMOUS_OWNED_BY_APP = 4
OBJECT_CREATION_TYPE_EPHEMERAL = 5

try:  # pragma: no cover
    from modal_proto.api_pb2 import MountGetOrCreateRequest  # type: ignore
except Exception:

    @dataclasses.dataclass
    class MountGetOrCreateRequest:  # type: ignore[no-redef]  (api.proto:2589-2596)
        deployment_name: str = ""
        namespace: int = 0
        environment_name: str = ""
        object_creation_type: int = OBJECT_CREATION_TYPE_UNSPECIFIED
        files: list = dataclasses.field(default_factory=list)
        app_id: str = ""


try:  # pragma: no cover
    from modal_proto.api_pb2 import (  # type: ignore
        MountFile, MountPutFileRequest, VolumePutFiles2Request, VolumePutFilesRequest)
except Exception:

    @dataclasses.dataclass
    class MountPutFileRequest:  # type: ignore[no-redef]  (api.proto:2607-2614)
        sha256_hex: str = ""
        data: bytes | None = None
        data_blob_id: str | None = None

        def WhichOneof(self, _name: str):
            return "data" if self.data is not None else ("data_blob_id" if self.data_blob_id else None)

    @dataclasses.dataclass
    class MountFile:  # type: ignore[no-redef]  (api.proto:2582-2587)
        filename: str = ""
        sha256_hex: str = ""
        mode: int = 0

    @dataclasses.dataclass
    class VolumePutFilesRequest:  # type: ignore[no-redef]
        volume_id: str = ""
        files: list = dataclasses.field(default_factory=list)
        disallow_overwrite_existing_files: bool = False

    class VolumePutFiles2Request:  # type: ignore[no-redef]  (api.proto:3954-3981)
        @dataclasses.dataclass
        class Block:
            contents_sha256: bytes = b""
            put_response: bytes | None = None

        @dataclasses.dataclass
        class File:
            path: str = ""
            mode: int = 0
            size: int = 0
            blocks: list = dataclasses.field(default_factory=list)

        def __init__(self, volume_id="", files=None, disallow_overwrite_existing_files=False):
            self.volume_id = volume_id
            self.files = files or []
            self.disallow_overwrite_existing_files = disallow_overwrite_existing_files


try:  # pragma: no cover
    from modal_proto.api_pb2 import VolumeGetFile2Request  # type: ignore
except Exception:

    @dataclasses.dataclass
    class VolumeGetFile2Request:  # type: ignore[no-redef]  (api.proto:3840-3845)
        volume_id: str = ""
        path: str = ""
        start: int = 0
        len: int = 0  # 0: to the end of the file


try:  # pragma: no cover
    from modal_proto.api_pb2 import SharedVolumeGetFileRequest, SharedVolumePutFileRequest  # type: ignore
except Exception:

    @dataclasses.dataclass
    class SharedVolumePutFileRequest:  # type: ignore[no-redef]  (api.proto:3555-3564)
        shared_volume_id: str = ""
        path: str = ""
        sha256_hex: str = ""
        data: bytes = b""
        data_blob_id: str = ""
        resumable: bool = False

    @dataclasses.dataclass
    class SharedVolumeGetFileRequest:  # type: ignore[no-redef]
        shared_volume_id: str = ""
        path: str = ""
