"""Where the time of one RoIAlign forward call goes at BASELINE cfg2, inside a CUDA graph as bench.py runs it.

    python tools/fwd_breakdown.py [--calls 120] [--sets 6]

Same inputs as bench.py (1x256x200x272 fp32, 512 RoIs, 7x7, sr=2, rotating input sets, seeds of rank 0), the forward
calls alone captured into one CUDA graph, replayed once to warm up and once under torch.profiler (CUDA activities).
Every call is cut out of the trace as the device operations (kernels and memsets) up to and including the main kernel;
reported per operation: mean device time and the mean gap to the previous operation of the same call (negative when
the two overlap, e.g. under programmatic dependent launch); per call: the time from its first operation's start to the
main kernel's start ("before_main_us") and to its end ("call_us").  On the stream path the main kernel includes its tail,
the in-place transpose of the output rows after a grid barrier (tools/stream_probe.py splits the two).  The card's name and
power limit are read in the same run.  Times taken under the profiler: use them for the split, not as a bench value.
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MAIN_KERNELS = ("roi_align_stream_fwd", "roi_align_strip_fwd", "roi_align_tiled", "roi_align_forward_generic")


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:  # noqa: BLE001
        return {"error": str(exc)}


def short_name(name):
    """'void b200::(anonymous namespace)::stream_prep<2>(...)' -> 'stream_prep'"""
    if "memset" in name.lower():
        return "memset"
    base = name.replace("(anonymous namespace)", "").split("(")[0].split("<")[0].strip()
    return base.split("::")[-1].split(" ")[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=120)
    ap.add_argument("--sets", type=int, default=6)
    args = ap.parse_args()
    import torch
    from detectron.pytorch_b200 import _lib
    from detectron.pytorch_b200 import synthetic as S
    if not torch.cuda.is_available():
        raise SystemExit("fwd_breakdown.py: no CUDA device")
    lib = _lib.load()
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    cfg = S.CFG2
    shape, P, scale, sr, R = cfg["shape"], cfg["pooled"], cfg["scale"], cfg["sampling_ratio"], cfg["rois"]
    N, C, H, W = shape
    nsets = max(2, args.sets)
    gen = torch.Generator(device=device); gen.manual_seed(1234)
    feats = [torch.randn(shape, generator=gen, device=device) for _ in range(nsets)]
    rois = [torch.from_numpy(S.make_rois(R, shape, scale, seed=i)).to(device) for i in range(nsets)]
    outs = [torch.empty((R, C, P, P), device=device) for _ in range(nsets)]
    ws_bytes = int(lib.b200_roi_align_workspace_bytes(N, R, H, W, P, P, sr))
    wss = [torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=device) for _ in range(nsets)]

    def fwd(i):
        j = i % nsets
        _lib.check(lib.b200_roi_align_forward_ws(feats[j].data_ptr(), scale, N, R, H, W, C, P, P, sr, rois[j].data_ptr(),
                                                 outs[j].data_ptr(), wss[j].data_ptr() if ws_bytes else None, ws_bytes,
                                                 torch.cuda.current_stream().cuda_stream), "fwd")

    for i in range(nsets):
        fwd(i)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fwd(0)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(args.calls):
            fwd(i)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); g.replay(); e1.record()
    torch.cuda.synchronize()
    graph_us = e0.elapsed_time(e1) * 1e3 / args.calls

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.replay()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    ops = [ev for ev in trace.get("traceEvents", [])
           if ev.get("ph") == "X" and ev.get("cat") in ("kernel", "gpu_memset")]
    ops.sort(key=lambda ev: float(ev["ts"]))

    calls, cur = [], []
    for ev in ops:
        cur.append(ev)
        if any(k in ev["name"] for k in MAIN_KERNELS):
            calls.append(cur)
            cur = []
    calls = calls[1:]                                         # the first call of the window has no predecessor to compare with
    dur = collections.defaultdict(list)
    gap = collections.defaultdict(list)
    before, span = [], []
    for call in calls:
        t0 = float(call[0]["ts"])
        for k, ev in enumerate(call):
            name = short_name(ev["name"])
            dur[name].append(float(ev["dur"]))
            if k > 0:
                prev = call[k - 1]
                gap[name].append(float(ev["ts"]) - (float(prev["ts"]) + float(prev["dur"])))
        main_ev = call[-1]
        before.append(float(main_ev["ts"]) - t0)
        span.append(float(main_ev["ts"]) + float(main_ev["dur"]) - t0)
    mean = lambda v: sum(v) / len(v) if v else None
    order = [short_name(ev["name"]) for ev in calls[0]] if calls else []
    result = {
        "card": card_info(),
        "workload": "RoIAlign forward 1x256x200x272 fp32, 512 RoIs, 7x7, sr=2; CUDA graph of %d calls, %d rotating sets" % (args.calls, nsets),
        "calls_traced": len(calls),
        "graph_us_per_call": graph_us,
        "ops": [{"op": n, "mean_us": mean(dur[n]), "gap_before_us": mean(gap[n])} for n in order],
        "before_main_us": mean(before),
        "call_us": mean(span),
        "note": "op times and gaps from torch.profiler (CUDA activities) over one graph replay; graph_us_per_call from CUDA events, profiler off",
    }
    print(json.dumps(result))
    return 0


if __name__ == "__main__":
    sys.exit(main())
