"""Stand-alone check + bandwidth probe of the NVLS all-reduce (csrc/nvls.cu) on N GPUs of one node:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29611 tools/test_nvls.py

Each rank fills a symmetric-memory fp32 buffer with rank-dependent values, runs barrier -> cb_nvls_allreduce_f32 -> barrier,
checks the average element-wise (bit-exact: the sums are small integers), then times the exchange of the two buffer sizes of a
training step (transformer 111.2 M, CNN 37.6 M elements incl. the frozen stem / res2 slots) against torch.distributed's NCCL all-reduce of the same buffers.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def main():
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    import torch.distributed._symmetric_memory as symm
    from clipbert_b200 import ops
    out = dict(world=world)
    for n in (4096, 37_610_688, 111_229_504):      # the CNN and transformer flat gradient buffers of the training step
        buf = symm.empty(n, dtype=torch.float32, device=dev)
        hdl = symm.rendezvous(buf, dist.group.WORLD)
        assert hdl.multicast_ptr, "no multicast mapping on this system"
        idx = torch.arange(n, device=dev, dtype=torch.float32) % 1024
        for ctas in (8, 32, 64):
            buf.copy_(idx * (rank + 1))
            hdl.barrier(channel=0)
            ops.nvls_allreduce(hdl.multicast_ptr, n, rank, world, 1.0 / world, ctas)
            hdl.barrier(channel=0)
            torch.cuda.synchronize()
            expect = idx * (sum(range(1, world + 1)) / world)
            ok = bool(torch.equal(buf, expect))
            # slice at an offset (the mid-backward bucket): elements [n/2, n) only
            buf.copy_(idx * (rank + 1))
            lo = (n // 2) // 64 * 64
            hdl.barrier(channel=0)
            ops.nvls_allreduce(hdl.multicast_ptr + 4 * lo, n - lo, rank, world, 1.0 / world, ctas)
            hdl.barrier(channel=0)
            torch.cuda.synchronize()
            ok = ok and bool(torch.equal(buf[lo:], expect[lo:])) and bool(torch.equal(buf[:lo], (idx * (rank + 1))[:lo]))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            dist.barrier()
            e0.record()
            for _ in range(10):
                hdl.barrier(channel=0)
                ops.nvls_allreduce(hdl.multicast_ptr, n, rank, world, 1.0 / world, ctas)
                hdl.barrier(channel=0)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 10
            out["n%d_ctas%d" % (n, ctas)] = dict(ok=ok, ms=round(ms, 4), bus_gbs=round(2 * (world - 1) / world * n * 4 / ms / 1e6, 1))
        ref = torch.zeros(n, device=dev)
        for _ in range(3):
            dist.all_reduce(ref, op=dist.ReduceOp.AVG)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            dist.all_reduce(ref, op=dist.ReduceOp.AVG)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        out["n%d_nccl" % n] = dict(ms=round(ms, 4), bus_gbs=round(2 * (world - 1) / world * n * 4 / ms / 1e6, 1))
    if rank == 0:
        print(json.dumps(out))
    dist.barrier()
    os._exit(0)


if __name__ == "__main__":
    main()
