"""Exceptions the host layer raises (names follow the reference's modal.exception)."""


class ExecutionError(Exception):
    """An upload step failed or an integrity check (ETag / digest comparison) did not hold."""


class ServiceError(Exception):
    """The server is temporarily unavailable (modal.exception.ServiceError)."""


class MountUploadTimeoutError(TimeoutError):
    """Raised when a Mount upload times out (modal.exception.MountUploadTimeoutError)."""
