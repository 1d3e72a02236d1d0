"""tools/pump_model.py -- the map pump on a machine WITHOUT a GPU: the real InputPreprocessor / InputPumper and bench.py's
null control plane around a stand-in for the hash call that behaves like b200h_hash_batch_host does towards Python:
it is entered through ctypes (GIL released), serialises the calls of one context on a mutex, holds a process-wide
"packing" mutex for PACK seconds per 4 096 payloads (the host's staging-copy capacity is one shared resource) and then
spends TAIL seconds on its own (last H2D chunk + kernel + D2H).  Everything is inside C, so the GIL traffic of the
real path is reproduced; the digests are zeros.  With PACK=0.030 TAIL=0.015 (33 GiB/s of packing, one measured host's
measured figure) the floor is 0.75 s per 100 000 x 256 KiB; the round-2 pump as measured on the box (1.04-1.12 s) comes
out at 1.01-1.07 s in this model, which is what makes it usable for host-side work when no GPU is at hand.

    PACK=0.030 TAIL=0.015 python tools/pump_model.py        # N=100000 inputs, 5 passes, min / median
"""
import ctypes
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import bench
from modal_client_b200 import _backend, blob_utils, parallel_map

C_SRC = r"""
#include <pthread.h>
#include <unistd.h>
static pthread_mutex_t pack = PTHREAD_MUTEX_INITIALIZER;
static pthread_mutex_t ctxmu[8] = {PTHREAD_MUTEX_INITIALIZER, PTHREAD_MUTEX_INITIALIZER, PTHREAD_MUTEX_INITIALIZER,
                                   PTHREAD_MUTEX_INITIALIZER, PTHREAD_MUTEX_INITIALIZER, PTHREAD_MUTEX_INITIALIZER,
                                   PTHREAD_MUTEX_INITIALIZER, PTHREAD_MUTEX_INITIALIZER};
void fake_hash(int ctx, int pack_us, int tail_us) {
    pthread_mutex_lock(&ctxmu[ctx & 7]);
    pthread_mutex_lock(&pack);
    usleep(pack_us);
    pthread_mutex_unlock(&pack);
    usleep(tail_us);
    pthread_mutex_unlock(&ctxmu[ctx & 7]);
}
"""
PACK = float(os.environ.get("PACK", "0.030"))
TAIL = float(os.environ.get("TAIL", "0.015"))
N = int(os.environ.get("N", 100_000))
tmp = tempfile.mkdtemp()
with open(os.path.join(tmp, "m.c"), "w") as f:
    f.write(C_SRC)
subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-o", os.path.join(tmp, "libm.so"), os.path.join(tmp, "m.c"), "-lpthread"])
LIB = ctypes.CDLL(os.path.join(tmp, "libm.so"))
LIB.fake_hash.argtypes = [ctypes.c_int] * 3


class StandInContext:
    device = -1
    made = 0

    def __init__(self):
        self.i = StandInContext.made
        StandInContext.made += 1

    def hash_buffers(self, bufs, flags=3):
        n = len(bufs)
        LIB.fake_hash(self.i, int(PACK * 1e6 * n / 4096), int(TAIL * 1e6))
        return np.zeros((n, 32), np.uint8), np.zeros((n, 16), np.uint8), np.zeros(n, np.uint64)


ctxs = [StandInContext() for _ in range(8)]
_backend.set_context(ctxs[0])
_backend.context_pool = lambda k: ctxs[:k]
blob_utils._upload_to_s3_url = bench._null_put
payloads = [bytes(262144)] * N
ts = []
for _ in range(5):
    stub = bench.NullStub()
    dt, batches, _tables = bench.run_map_pump(payloads, stub)
    ts.append(dt)
print(f"{N} inputs, {batches} windows, {parallel_map.HASH_WINDOWS_IN_FLIGHT} in flight; packing floor {PACK * batches:.2f} s: "
      f"step min {min(ts):.3f} s, median {sorted(ts)[2]:.3f} s; stages of the last pass {bench.run_map_pump.last_stats}")
