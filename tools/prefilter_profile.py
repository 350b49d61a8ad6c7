#!/usr/bin/env python
"""prefilter_profile.py [rows] [dim] — torch.profiler kernel times of single-query searches on one synthetic cosine storage (generated on the
device, as prefilter_probe.py), for each first stage of the 6-bit plane's scan (option prefilter_stage1: 5 = the 5-bit codes, 0 = the
block-scaled 4-bit plane); prints one JSON line with the mean time per search of every kernel and the stage-1 bytes over its time."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

from qdrant_b200 import scorer as qb
from qdrant_b200._capi import check, lib, vp

rows = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
dim = int(sys.argv[2]) if len(sys.argv) > 2 else 768
dev = torch.device("cuda", 0)
st = qb.DenseVectorStorage(None, qb.Distance.Cosine, count=rows, dim=dim, device=0)
gen = torch.Generator(device=dev); gen.manual_seed(42)
for r0 in range(0, rows, 500_000):
    n = min(500_000, rows - r0)
    x = torch.randn((n, dim), generator=gen, device=dev, dtype=torch.float32)
    check(lib().qb_metric_preprocess_device(0, int(qb.Distance.Cosine), dim, n, vp(x.data_ptr()), dim * 4))
    st.write_rows_device(r0, n, x.data_ptr(), dim * 4)
    del x
torch.cuda.synchronize()
queries = torch.from_numpy(np.random.default_rng(43).standard_normal((16, dim)).astype(np.float32)).to(dev)
d_out = torch.empty((1, 10), dtype=torch.int64, device=dev); d_cnt = torch.empty((1,), dtype=torch.int32, device=dev)
d_pad = (dim + 31) // 32 * 32
stride = {5: (5 * d_pad // 8 + 12 + 7) // 8 * 8, 0: ((d_pad // 2 + d_pad // 16 + 3) // 4 * 4 + 8 + 7) // 8 * 8}
K = 32
out = {"rows": rows, "dim": dim, "card": torch.cuda.get_device_name(0)}
for stage1 in (5, 0):
    qb.set_option("prefilter_stage1", stage1)
    step = lambda i: check(lib().qb_search_batch_device(st._h, vp(queries[i % 16].data_ptr()), 1, 10, vp(d_out.data_ptr()), vp(d_cnt.data_ptr())))
    for i in range(8):
        step(i)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(K):
            step(i)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name.replace("(anonymous namespace)::", "").replace("void ", "").split("<")[0].split("(")[0]
            kern[name] = kern.get(name, 0.0) + e.device_time_total / 1e3 / K
    s1 = kern.get("dense_q4b_filter_kernel" if stage1 == 0 else "dense_q5_filter_kernel", 0.0)
    out[f"stage1_{stage1}"] = {"kernel_ms_per_search": {k: round(v, 4) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])},
                               "stage1_bytes": rows * stride[stage1], "stage1_TBps": rows * stride[stage1] / (s1 * 1e-3) / 1e12 if s1 else None}
qb.set_option("prefilter_stage1", 0)
out["fallbacks"] = int(st.search_stats()[1])
print(json.dumps(out))
