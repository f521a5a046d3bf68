import os, sys, traceback
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch, torch.multiprocessing as mp
from slab_cases import collect, free_port, slab_worker

if __name__ == "__main__":
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=slab_worker, args=(r, 2, port, 48, 2, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = collect(procs, q, 100)
    for r in res:
        print(r[0], r[1][-3000:])
    print("n results", len(res))
