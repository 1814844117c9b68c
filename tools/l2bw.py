"""L2 read bandwidth of this card (what a kernel that streams L2-resident data, such as the weight rings of
mlp_sa_fact2w_kernel and mlp_fp2_kernel, can be held against): buffers of 8-24 MB (H100: 50 MB of L2) read by
`reps` sum reductions captured in one CUDA graph, CUDA events around each replay, the median of five replays.
Prints one JSON line with the device name and GB/s per buffer size."""
import json
import statistics

import torch

dev = torch.device("cuda:0")
reps = 200


def read_rate(mb):
    n = mb * (1 << 20) // 4
    a = torch.ones(n, dtype=torch.float32, device=dev)
    r = torch.empty((), dtype=torch.float32, device=dev)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):   # warm-up outside the capture (the reduction picks its launch shape here)
        for _ in range(3):
            torch.sum(a, dim=0, out=r)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            torch.sum(a, dim=0, out=r)
    g.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e-3 / reps)
    assert float(r) == float(n)
    return 4 * n / statistics.median(times) / 1e9


out = {"gpu": torch.cuda.get_device_name(dev)}
for mb in (8, 16, 24):
    out[f"read_{mb}MB_GBps"] = round(read_rate(mb), 1)
print(json.dumps(out))
