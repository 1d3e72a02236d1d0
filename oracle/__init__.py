"""oracle/ -- TEST INFRASTRUCTURE ONLY (CPU checker for the GPU hash path).

Nothing under ``modal_client_b200/`` may import this package.  Allowed users:
``tests/``, ``__graft_entry__.smoke()``, ``oracle/gen_golden.py`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs.

Two independent CPU statements of the reference's path live here:

* ``oracle.c_oracle``  -- ctypes binding of ``liboracle.so`` (``hash_oracle.c``): a from-the-spec
  scalar SHA-256 (FIPS 180-4) / MD5 (RFC 1321) plus the trimmed-block and multipart-ETag helpers.
* ``oracle.ref_port``  -- a Python restatement of the reference's *control flow*
  (``hash_utils._update`` / ``get_upload_hashes`` / ``_find_end_of_block`` / ``_gather_block`` /
  multipart ETag) on top of ``hashlib`` -- the very library the reference calls
  (``py/modal/_utils/hash_utils.py:34,42,50,75,78`` of the original project).

Parity pinning: see ``tests/test_oracle.py`` (NIST / RFC known answers, hashlib cross-check,
and ``tests/golden/*.json`` recorded from the unmodified original project by ``oracle/gen_golden.py``).
"""
