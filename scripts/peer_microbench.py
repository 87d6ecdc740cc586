"""NVLink access-pattern micro-benchmark for the peer-memory sparse step (2+ GPUs):
    torchrun --nproc-per-node 2 scripts/peer_microbench.py
Random 64-B row reads from the peer, random 64-B row writes to the peer, contiguous peer reads / writes; rank 0 drives,
the peer idles (its buffers stay mapped).  Prints GB/s per pattern (CUDA events, best of 5)."""
import ctypes
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dev = torch.device("cuda", torch.cuda.current_device())
    dist.init_process_group("nccl", device_id=dev)
    from torcheasyrec_b200.peer_exchange import _Symm

    L = ctypes.CDLL(os.path.join(ROOT, "scripts", "libtzk_peer_bench.so"))
    P, I64, I32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32
    L.bench_rand_read64.argtypes = [P, P, I64, P, I32, I32, P]
    L.bench_rand_write64.argtypes = [P, P, I64, P, I32, P]
    L.bench_seq_copy.argtypes = [P, I64, P, I32, P]
    L.bench_rand_read64_mixed.argtypes = [P, P, P, I64, P, I32, P]
    rows = int(os.environ.get("ROWS_M", "16")) * 1024 * 1024       # 64-B rows per rank (16 M = 1 GiB)
    tab = _Symm(rows * 16, torch.float32, dev, dist.group.WORLD)
    tab.t.normal_()
    torch.cuda.synchronize()
    dist.barrier()
    if rank == 0:
        peer = int(tab.ptrs[1 % world])
        mine = int(tab.ptrs[0])
        n = 851968                              # 26 * 65536 / 2 rows = the remote half of one gather at N = 2
        idx = torch.randint(0, rows, (n,), device=dev, dtype=torch.int32)
        loc = torch.empty(n * 16, device=dev)
        st = torch.cuda.current_stream().cuda_stream

        def timed(fn, reps=5):
            best = 1e9
            for _ in range(reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                best = min(best, e0.elapsed_time(e1))
            return best

        gb = n * 64 / 1e9
        print(f"region: {rows * 64 / 2 ** 30:.1f} GiB per rank", flush=True)
        n2 = 2 * n                              # a whole N = 2 gather: half of the rows local, half on the peer
        idx2 = torch.randint(0, rows, (n2,), device=dev, dtype=torch.int32)
        loc2 = torch.empty(n2 * 16, device=dev)
        for grid in (132 * 4, 132 * 8):
            ms = timed(lambda: L.bench_rand_read64_mixed(mine, peer, idx2.data_ptr(), n2, loc2.data_ptr(), grid, st))
            print(f"rand_read64  MIXED local/peer in every warp, {n2} rows grid={grid:<5} {ms * 1e3:8.1f} us  "
                  f"(peer half: {gb / ms * 1e3:7.1f} GB/s)", flush=True)
        for U in (1, 8):
            for grid in (132, 132 * 8):
                ms = timed(lambda: L.bench_rand_read64(peer, idx.data_ptr(), n, loc.data_ptr(), U, grid, st))
                print(f"rand_read64  peer  U={U:<2} grid={grid:<5} {ms * 1e3:8.1f} us  {gb / ms * 1e3:7.1f} GB/s", flush=True)
        ms = timed(lambda: L.bench_rand_read64(mine, idx.data_ptr(), n, loc.data_ptr(), 8, 132 * 8, st))
        print(f"rand_read64  LOCAL U=8  grid=1184  {ms * 1e3:8.1f} us  {gb / ms * 1e3:7.1f} GB/s", flush=True)
        for grid in (132, 132 * 4, 132 * 8, 132 * 16):
            ms = timed(lambda: L.bench_rand_write64(loc.data_ptr(), idx.data_ptr(), n, peer, grid, st))
            print(f"rand_write64 peer       grid={grid:<5} {ms * 1e3:8.1f} us  {gb / ms * 1e3:7.1f} GB/s", flush=True)
        ms = timed(lambda: L.bench_rand_write64(loc.data_ptr(), idx.data_ptr(), n, mine, 132 * 8, st))
        print(f"rand_write64 LOCAL      grid=1184  {ms * 1e3:8.1f} us  {gb / ms * 1e3:7.1f} GB/s", flush=True)
        nf = 64 * 1024 * 1024                   # 256 MB contiguous
        big = torch.empty(nf, device=dev)
        for grid in (132 * 4, 132 * 16):
            ms = timed(lambda: L.bench_seq_copy(peer, nf, big.data_ptr(), grid, st))
            print(f"seq read  peer->local   grid={grid:<5} {ms * 1e3:8.1f} us  {nf * 4 / 1e9 / ms * 1e3:7.1f} GB/s", flush=True)
            ms = timed(lambda: L.bench_seq_copy(big.data_ptr(), nf, peer, grid, st))
            print(f"seq write local->peer   grid={grid:<5} {ms * 1e3:8.1f} us  {nf * 4 / 1e9 / ms * 1e3:7.1f} GB/s", flush=True)
    torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
