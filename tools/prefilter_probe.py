#!/usr/bin/env python
"""prefilter_probe.py [rows] [dim] — single-query searches over one synthetic cosine storage (generated on the device), device-timed, for several
ring-slot sizes / producer-warp counts of the shadow-plane filter kernels and the three planes; prints one JSON line.  Results of every variant are compared with the exact scan.
"candidates" counts, per query, the rows each integer plane's bound lets through (the kernels' bounds restated in torch on the same rows, f64 where they round up):
on the 6-bit plane, for each candidate size of its threshold sample (n / 16, n / 8, n / 4 rows), the rows of the 5-bit first stage (q6_stage1), those of
them the 6-bit test keeps (q6_stage2) and the rows of the block-scaled 4-bit first stage (q4b_stage1, the default), with the threshold restated as the exact top-k of the prefix (the kernel ranks the prefix by its approximate score
first, so its threshold can only be lower, by the ranking error); on the int8 plane, with the f32 sample of 1/64 of the rows it keeps."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

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
queries = np.random.default_rng(43).standard_normal((16, dim)).astype(np.float32)
d_q = torch.from_numpy(queries).to(dev)
d_out = torch.empty((1, 10), dtype=torch.int64, device=dev); d_cnt = torch.empty((1,), dtype=torch.int32, device=dev)
stream = torch.cuda.ExternalStream(st.stream_ptr(), device=dev)


def run(K=30):
    def step(i):
        check(lib().qb_search_batch_device(st._h, vp(d_q[i % 16].data_ptr()), 1, 10, vp(d_out.data_ptr()), vp(d_cnt.data_ptr())))
    for i in range(5):
        step(i)
    torch.cuda.synchronize()
    st.profile_read(reset=True); st.profile(True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for i in range(K):
        step(i)
    e1.record(stream)
    torch.cuda.synchronize()
    n_prof, prof_ms = st.profile_read(reset=True); st.profile(False)
    return {"ms_per_step": e0.elapsed_time(e1) / K, "qps": K / (e0.elapsed_time(e1) / 1e3), "kernel_ms": prof_ms / max(n_prof, 1)}


qb.set_option("disable_prefilter", 1)
exact = [st.search_batch(queries[i], 10)[0] for i in range(4)]
out = {"rows": rows, "dim": dim, "exact_f32_scan": run(10)}
qb.set_option("disable_prefilter", 0)
for plane, name in ((0, "q6"), (2, "int8"), (1, "bf16")):
    qb.set_option("prefilter_plane", plane)
    for prod in (1, 2, 4):
        qb.set_option("prefilter_producers", prod)
        for slot in (12288, 8192, 6144):
            qb.set_option("prefilter_slot_bytes", slot)
            got = [st.search_batch(queries[i], 10)[0] for i in range(4)]
            same = all(np.array_equal(a["idx"], b["idx"]) and np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32)) for a, b in zip(got, exact))
            r = run()
            r["identical_to_exact_scan"] = bool(same)
            out[f"{name}_producers{prod}_slot{slot}"] = r
qb.set_option("prefilter_producers", 0)
qb.set_option("prefilter_slot_bytes", 0); qb.set_option("prefilter_plane", 0)
out["fallbacks"] = int(st.search_stats()[1])


def candidate_counts(nq=16, top=10):
    """Rows with upper bound >= thr_q - slack_q on the 6-bit plane's two stages (per prefix size) and the int8 plane, thr_q = the exact top-`top`
    score of the sample prefix."""
    qd = torch.from_numpy(queries[:nq]).to(dev).double()
    qd = (qd / qd.norm(dim=1, keepdim=True)).float().double()          # cosine queries are normalised
    qmax = qd.abs().amax(1, keepdim=True)
    sq = (qmax / 127).float().double()
    y = (qd * (127 / qmax)).float().double()
    h = y.round().clamp(-127, 127)
    l = ((y - h) * 254).round().clamp(-127, 127)
    q1, qn = qd.abs().sum(1), qd.norm(dim=1)
    prefixes = {"n/16": rows // 16, "n/8": rows // 8, "n/4": rows // 4}
    sample8 = min(131072, max(16384, rows // 64))
    e1 = q1 * (0.5 + 2.0 ** -13) + sq[:, 0] * dim * 0.066
    e1_5 = q1 * (1 + 2.0 ** -13) + sq[:, 0] * dim * 0.066
    e2 = sq[:, 0] * dim ** 0.5 * 0.00202
    e8 = q1 * (0.5 + 2.0 ** -13) + sq[:, 0] * dim * 0.27
    g = torch.Generator(device=dev)

    def chunks():
        g.manual_seed(42)
        for r0 in range(0, rows, 500_000):
            n = min(500_000, rows - r0)
            x = torch.randn((n, dim), generator=g, device=dev, dtype=torch.float32)
            check(lib().qb_metric_preprocess_device(0, int(qb.Distance.Cosine), dim, n, vp(x.data_ptr()), dim * 4))
            yield r0, n, x

    # pass 1: max row norm, and the exact top-`top` of every prefix
    mxn, best = 0.0, {k: None for k in prefixes}
    for r0, n, x in chunks():
        mxn = max(mxn, float(x.double().norm(dim=1).max()))
        for k, p in prefixes.items():
            if r0 < p:
                s = x[: p - r0].double() @ qd.T
                best[k] = s if best[k] is None else torch.cat([best[k], s])
                best[k] = best[k].topk(top, dim=0).values
        if r0 == 0:
            thr8 = (x[:sample8].double() @ qd.T).topk(top, dim=0).values[-1]
    thr = {k: v[-1] for k, v in best.items()}
    slack6 = 2 * (dim * 2.0 ** -22 + 2.0 ** -17) * qn * mxn
    slack8 = (dim * 2.0 ** -22 + 2.0 ** -17) * (1 + dim ** 0.5 / 127) * qn * mxn
    c5 = {k: torch.zeros(nq, dtype=torch.int64, device=dev) for k in prefixes}
    c6 = {k: torch.zeros(nq, dtype=torch.int64, device=dev) for k in prefixes}
    c8 = torch.zeros(nq, dtype=torch.int64, device=dev)
    c4b = {k: torch.zeros(nq, dtype=torch.int64, device=dev) for k in prefixes}
    # pass 2: the bounds of every row against each threshold
    for r0, n, x in chunks():
        mx = x.abs().amax(1, keepdim=True)
        sr = (mx / 31).double()
        c = (x * (31 / mx)).round().clamp(-31, 31).double()
        rho = (x.double() - sr * c).norm(dim=1, keepdim=True)
        up6 = sr * sq.T * (c @ h.T + (c @ l.T) / 254) + torch.minimum(sr * e1, rho * (qn + e2) + e2 * mxn)
        c5c = 2 * torch.div(c + 31, 2, rounding_mode="floor") + 0.5 - 31      # the 5-bit code's reconstruction
        rho5 = (x.double() - sr * c5c).norm(dim=1, keepdim=True)
        up5 = sr * sq.T * (c5c @ h.T + (c5c @ l.T) / 254) + torch.minimum(sr * e1_5, rho5 * (qn + e2) + e2 * mxn)
        # the block-scaled 4-bit stage (dense_q4b_filter_kernel): k_b per 16 dims, codes in [-7, 7], bound approx + min(t1, t2) + ev
        nb = -(-dim // 16)
        xp = torch.nn.functional.pad(x, (0, nb * 16 - dim)).view(n, nb, 16)
        s4 = (mx / 7).double()
        kb = torch.where(xp.abs().amax(2) > 0, torch.ceil(xp.abs().amax(2) * (255 / mx)).clamp(1, 255), torch.zeros((), device=dev)).double()
        sb = s4 * kb / 255
        cb = torch.where(sb[:, :, None] > 0, (xp.double() / sb[:, :, None]).round().clamp(-7, 7), torch.zeros((), device=dev, dtype=torch.float64))
        xh = (sb[:, :, None] * cb).view(n, nb * 16)[:, :dim]
        rho4 = (x.double() - xh).norm(dim=1, keepdim=True)
        eb = torch.nn.functional.pad(qd.abs(), (0, nb * 16 - dim)).view(nq, nb, 16).sum(2) * (0.5 + 2.0 ** -13) \
            + sq * 0.014 * torch.clamp(dim - 16 * torch.arange(nb, device=dev), 0, 16)
        up4 = xh @ (sq * (h + l / 254)).T + torch.minimum(sb @ eb.T, rho4 * (qn + e2) + e2 * mxn) + 2.0 ** -19 * (qn + e2) * (mxn + rho4)
        for k in prefixes:
            p5 = up5 >= thr[k] - slack6
            c5[k] += p5.sum(0)
            c6[k] += (p5 & (up6 >= thr[k] - slack6)).sum(0)
            c4b[k] += (up4 >= thr[k] - slack6).sum(0)
        s8 = (mx / 127).double()
        c = (x * (127 / mx)).round().clamp(-127, 127).double()
        up8 = s8 * (sq.T * (c @ h.T + (c @ l.T) / 254) + e8)
        c8 += (up8 >= thr8 - slack8).sum(0)
        del x, c, rho, up6, up8, c5c, rho5, up5, xp, cb, xh, up4
    return {"q6": {k: {"sample_rows": prefixes[k], "q6_stage1": c5[k].tolist(), "q6_stage2": c6[k].tolist(),
                  "q4b_stage1": c4b[k].tolist()} for k in prefixes},
            "int8": c8.tolist(), "int8_sample_rows": sample8}


st.close()
torch.cuda.empty_cache()
out["candidates"] = candidate_counts()
print(json.dumps(out))
