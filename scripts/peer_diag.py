"""diagnostic: which kinds of access to a CUDA-IPC peer buffer work from this process's kernels"""
import ctypes as C, os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl")
from tinysql_b200 import _lib as L
lib = L.load(); L.check(lib.tq_init(local))
dev = torch.device("cuda", local)
own = C.c_void_p(); L.check(lib.tq_device_alloc(8 << 20, C.byref(own))); L.check(lib.tq_memset_device(own, 0, 8 << 20))
hb = (C.c_ubyte * 64)(); L.check(lib.tq_ipc_get_handle(own, hb))
g = [None] * world
dist.all_gather_object(g, bytes(hb))
peer = (rank + 1) % world
pp = C.c_void_p(); L.check(lib.tq_ipc_open_handle((C.c_ubyte * 64).from_buffer_copy(g[peer]), C.byref(pp)))
class PT:
    def data_ptr(self): return pp.value
pt = PT()
print(rank, "peer ptr", hex(pp.value), flush=True)
def step(name, f):
    try:
        f(); lib.tq_device_synchronize(); torch.cuda.synchronize()
        print(rank, name, "OK", flush=True)
    except Exception as e:
        print(rank, name, "FAILED", str(e)[:200], flush=True); raise
step("memset peer via lib", lambda: L.check(lib.tq_memset_device(C.c_void_p(pt.data_ptr()), 1, 64)))
dist.barrier()
# one region push of 10000 rows into 2 destinations: this rank's own buffer (destination 0) and the peer's (destination 1).
# Every buffer holds a {rows, epoch} slot per source at its start and, from byte 4096, 2 region columns of CAP rows per source.
CAP = 20000
slot_of = lambda base, src: base + 16 * src
region_of = lambda base, src, c: base + 4096 + (src * 2 + c) * CAP * 8
k = torch.arange(10000, dtype=torch.int64, device=dev); v = k * 2
def push():
    cols = (L.TQColumn * 2)()
    for i, t in enumerate((k, v)):
        cols[i].length, cols[i].data, cols[i].null_bitmap, cols[i].offsets = 10000, t.data_ptr(), None, None
    dest = (C.c_void_p * 4)(*[region_of(b, rank, c) for b in (own.value, pp.value) for c in range(2)])
    cnts = (C.c_void_p * 2)(slot_of(own.value, rank), slot_of(pp.value, rank))
    L.check(lib.tq_partition_push_regions(2, cols, 0, 10000, 2, None, 0, dest, cnts, CAP, None, None, 0, 0, 1))
    L.check(lib.tq_partition_push_sync(0))
step("region push, destination 1 = peer", push)
dist.barrier()
src = (rank - 1) % world   # the rank whose destination 1 is this rank
hostslot = np.zeros(2, np.uint64); L.check(lib.tq_memcpy_d2h(hostslot.ctypes.data, C.c_void_p(slot_of(own.value, src)), 16))
rows = int(hostslot[0]); received = np.zeros(2 * CAP, np.int64)
L.check(lib.tq_memcpy_d2h(received.ctypes.data, C.c_void_p(region_of(own.value, src, 0)), 2 * CAP * 8))
print(rank, "received from", src, "rows", rows, "epoch", int(hostslot[1]), "sum", int(received[:rows].sum() + received[CAP:CAP + rows].sum()), flush=True)
dist.destroy_process_group()
