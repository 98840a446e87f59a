"""N -> 1 peer-write probe (round-2 tool): how fast can ranks 1..N-1 push into ONE GPU's memory over NVLink while that
GPU is idle?  Run under torchrun at 2, 4, 8 GPUs:

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 scripts/peer_probe.py

Every rank copies a 2 GiB local buffer into its slice of a buffer that rank 0 allocated and exported through CUDA IPC
(rtcb200PeerAlloc/Export/Import, the same plumbing the hit gather uses); the aggregate rate into rank 0 is printed for
1 .. N-1 concurrent senders, to compare with the rate at which rank 0 receives the hit gather of a multi-GPU bench run."""
import ctypes as C
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import embree_b200  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    lib = embree_b200.load()
    dev = lib.new_device(f"gpu={local}")
    nbytes = 2 << 30
    handle = [None]
    if rank == 0:
        gbuf = lib.rtcb200PeerAlloc(dev, world * nbytes)
        h64 = (C.c_ubyte * 64)()
        assert lib.rtcb200PeerExport(dev, C.c_void_p(gbuf), h64) == 0
        handle = [bytes(h64)]
    dist.broadcast_object_list(handle, src=0)
    if rank != 0:
        gbuf = lib.rtcb200PeerImport(dev, (C.c_ubyte * 64).from_buffer_copy(handle[0]))
    lib.check(dev)
    src = torch.ones(nbytes // 4, dtype=torch.float32, device=f"cuda:{local}")
    flag = torch.zeros(1, device=f"cuda:{local}")
    for senders in range(1, world):
        times = []
        for it in range(4):
            dist.barrier()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if 1 <= rank <= senders:
                lib.rtcb200PeerCopy(dev, C.c_void_p(gbuf + rank * nbytes), C.c_void_p(src.data_ptr()), nbytes)
            e1.record()
            torch.cuda.synchronize()
            ms = torch.tensor([e0.elapsed_time(e1)], device=f"cuda:{local}")
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            times.append(float(ms.item()))
        if rank == 0:
            best = min(times[1:])
            print(f"{senders} sender(s) -> rank 0: {senders * nbytes / best * 1e-6:8.1f} GB/s aggregate ({best:.2f} ms for {senders} x 2 GiB)", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
