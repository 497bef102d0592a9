"""Where the streaming RoIAlign forward's main kernel (roi_align_stream_fwd) spends its time, at BASELINE cfg2 in a CUDA graph.

    python tools/stream_probe.py [--calls 60] [--sets 6] [--src PATH] [--out FILE] [--keep DIR]

The library carries no instrumentation.  This tool copies csrc/roi_align_stream.cu (or --src), inserts time stamps at fixed
anchors of the main kernel (every anchor must match exactly once, else the tool stops), compiles the copy on its own into a
small shared library with nvcc (same flags as the library) and runs clear -> prep -> main through it, the calls captured in one
CUDA graph with rotating input sets as bench.py and tools/fwd_breakdown.py run them.  Every warp of every CTA writes one record
of the last call:

  CTA      globaltimer after griddepcontrol.wait, at the warp's end of the fragment loop, after the grid barrier and at the
           end of the tail (the in-place transpose of the output rows)
  producer clock64 cycles blocked in mbar_wait(empty) -- the ring full, consumers holding slots; rows of the stream
  consumer clock64 cycles blocked on rows it only passes through (acquire_to before a fragment's key and at an item's tail),
           blocked on the rows of a fragment (acquire_to(end)), in the bin loop (its output stores included); fragments and
           bins it computed

"main_loop" is the span from the first CTA's start to the last warp's end of the fragment loop; "tail" the span from there
to the last warp's end of the transpose (grid barrier included).  Cycle shares are per warp (its own clock64 lifetime up to the
end of the fragment loop), averaged over the warps of a class; the per-CTA columns use globaltimer.  The stamps cost a few
instructions per row and per fragment: compare the probed kernel's span with the uninstrumented one (tools/fwd_breakdown.py)
before reading absolute numbers from it.  The card's name and power limit are read in the same run.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from detectron.pytorch_b200 import build as B  # noqa: E402

NREC = 14                                                     # u64 per warp record
WARPS = 20                                                    # 16 consumer + 4 producer warps per CTA

# (anchor, replacement): the replacement keeps the anchor text and adds the stamps around it
PATCHES = [
    ("__device__ u64* g_stream_dead = nullptr;\n",
     "__device__ u64* g_stream_dead = nullptr;\n"
     "__device__ u64* g_probe = nullptr;                         // [CTA][20 warps][14] records of the last call\n"
     "__device__ __forceinline__ u64 probe_gtime() { u64 t; asm volatile(\"mov.u64 %0, %globaltimer;\" : \"=l\"(t)); return t; }\n"),
    ("    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;\n\n    if (warp >= kConsumerWarps) {\n",
     "    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;\n"
     "    const u64 pr_g0 = probe_gtime();\n"
     "    const long long pr_c0 = clock64();\n"
     "    long long pr_w0 = 0, pr_w1 = 0, pr_comp = 0;\n"
     "    unsigned pr_n0 = 0, pr_n1 = 0, pr_n2 = 0;\n"
     "    auto pr_write = [&]() {\n"
     "        if (g_probe == nullptr || lane != 0) return;\n"
     "        u64* rec = g_probe + ((size_t)blockIdx.x * 20 + warp) * 14;\n"
     "        rec[0] = pr_g0; rec[1] = probe_gtime(); rec[2] = (u64)(clock64() - pr_c0);\n"
     "        rec[3] = (u64)pr_w0; rec[4] = (u64)pr_w1; rec[5] = (u64)pr_comp;\n"
     "        rec[6] = pr_n0; rec[7] = pr_n1; rec[8] = pr_n2; rec[9] = (u64)(L1 - L0); rec[11] = 1;\n"
     "    };\n\n"
     "    if (warp >= kConsumerWarps) {\n"),
    # producer: blocked on a free slot; rows staged / rows of the stream
    ("                mbar_wait(empty, (ephase >> slot) & 1u, 0x1000u + (unsigned)y);\n",
     "                { const long long pc = clock64(); mbar_wait(empty, (ephase >> slot) & 1u, 0x1000u + (unsigned)y); pr_w0 += clock64() - pc; }\n"
     "                ++pr_n1;\n"),
    ("        }\n        return;\n    }\n",
     "        }\n        pr_write();\n        return;\n    }\n"),
    # consumer: pass-through waits, fragment waits, bin loop (stores included)
    ("                acquire_to(acq + 1, 0x2000u);\n",
     "                { const long long pc = clock64(); acquire_to(acq + 1, 0x2000u); pr_w0 += clock64() - pc; }\n"),
    ("            acquire_to(end, 0x2800u);                           // rows [key, end) must be resident\n",
     "            { const long long pc = clock64(); acquire_to(end, 0x2800u); pr_w1 += clock64() - pc; }\n"
     "            const long long pr_cc = clock64(); ++pr_n0; pr_n1 += npw;\n"),
    ("            __syncwarp();                                       // the table buffer is rewritten for the next fragment\n",
     "            __syncwarp();                                       // the table buffer is rewritten for the next fragment\n"
     "            pr_comp += clock64() - pr_cc;\n"),
    ("            acquire_to(acq + 1, 0x3000u);\n",
     "            { const long long pc = clock64(); acquire_to(acq + 1, 0x3000u); pr_w0 += clock64() - pc; }\n"),
    ("            release_to(acq);\n        }\n        __syncwarp();\n    }\n}\n",
     "            release_to(acq);\n        }\n        __syncwarp();\n        ++pr_n2;\n    }\n    pr_write();\n}\n"),
    # tail: after the grid barrier, and at the end of the transpose
    ("    prepass::grid_barrier(a.ticket);\n",
     "    prepass::grid_barrier(a.ticket);\n"
     "    const u64 pr_t1 = probe_gtime();\n"),
    ("    else transpose_rows<1>(a, blocks);\n}\n",
     "    else transpose_rows<1>(a, blocks);\n"
     "    if (g_probe != nullptr && (threadIdx.x & 31) == 0) {\n"
     "        u64* rec = g_probe + ((size_t)blockIdx.x * 20 + (threadIdx.x >> 5)) * 14;\n"
     "        rec[12] = pr_t1; rec[13] = probe_gtime();\n"
     "    }\n}\n"),
]

ENTRY = r"""
namespace b200 { unsigned long long g_launch_count = 0; }     // the library defines it in api.cu
extern "C" __attribute__((visibility("default"))) int probe_forward(const float* bottom, float scale, int N, int R, int H, int W, int C,
        int PH, int PW, int sr, const float* rois, float* top, void* ws, size_t ws_bytes, cudaStream_t stream) {
    return b200::roi_align_forward_stream(bottom, scale, N, R, H, W, C, PH, PW, sr, rois, top, nullptr, ws, ws_bytes, stream);
}
extern "C" __attribute__((visibility("default"))) size_t probe_ws_bytes(int N, int R, int H, int W, int PH, int PW, int sr) {
    return b200::roi_align_stream_workspace_bytes(N, R, H, W, PH, PW, sr);
}
extern "C" __attribute__((visibility("default"))) int probe_set(unsigned long long* p) {
    return (int)cudaMemcpyToSymbol(b200::g_probe, &p, sizeof(p));
}
"""


def patched_source(src):
    for anchor, repl in PATCHES:
        n = src.count(anchor)
        if n != 1:
            raise SystemExit("stream_probe.py: anchor found %d times (want 1): %r" % (n, anchor[:80]))
        src = src.replace(anchor, repl)
    return src + ENTRY


def build_probe(src_path, workdir):
    with open(src_path) as f:
        src = patched_source(f.read())
    cu = os.path.join(workdir, "roi_align_stream_probe.cu")
    with open(cu, "w") as f:
        f.write(src)
    so = os.path.join(workdir, "libstream_probe.so")
    nvcc = B.find_nvcc()
    if nvcc is None:
        raise SystemExit("stream_probe.py: nvcc not found")
    cmd = [nvcc] + B.NVCC_FLAGS + ["-Xptxas", "-v", "-I", B.CSRC, "-I", B.INCLUDE, "-o", so, cu]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout)
        raise SystemExit("stream_probe.py: nvcc failed (exit %d)" % res.returncode)
    return so, res.stdout


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:  # noqa: BLE001
        return {"error": str(exc)}


def summarize(rec, ctas):
    """rec: [ctas][20][14] u64 of one call -> the breakdown table."""
    med = statistics.median
    t0 = min(int(rec[c][w][0]) for c in range(ctas) for w in range(WARPS))
    cta_start, cta_end, cta_rows, cta_frags, cta_bins = [], [], [], [], []
    prod_wait, cons_pass, cons_frag, cons_comp = [], [], [], []
    for c in range(ctas):
        cta_start.append((int(rec[c][0][0]) - t0) / 1e3)
        cta_end.append((max(int(rec[c][w][1]) for w in range(WARPS)) - t0) / 1e3)
        cta_rows.append(sum(int(rec[c][w][7]) for w in range(16, WARPS)) // 4)
        cta_frags.append(sum(int(rec[c][w][6]) for w in range(16)))
        cta_bins.append(sum(int(rec[c][w][7]) for w in range(16)))
        for w in range(WARPS):
            life = max(1, int(rec[c][w][2]))
            if w >= 16:
                prod_wait.append(int(rec[c][w][3]) / life)
            else:
                cons_pass.append(int(rec[c][w][3]) / life)
                cons_frag.append(int(rec[c][w][4]) / life)
                cons_comp.append(int(rec[c][w][5]) / life)
    cta_time = [e - s for s, e in zip(cta_start, cta_end)]
    main_end = max(cta_end)
    barrier_out = (max(int(rec[c][w][12]) for c in range(ctas) for w in range(WARPS)) - t0) / 1e3
    tail_end = (max(int(rec[c][w][13]) for c in range(ctas) for w in range(WARPS)) - t0) / 1e3
    mean = lambda v: sum(v) / len(v)
    order = sorted(range(ctas), key=lambda c: cta_time[c])
    return {
        "span_us": tail_end - min(cta_start),
        "main_loop_span_us": main_end - min(cta_start),
        "tail_span_us": tail_end - main_end,
        "last_barrier_exit_after_main_loop_us": barrier_out - main_end,
        "cta_time_us": {"max": max(cta_time), "median": med(cta_time), "min": min(cta_time)},
        "cta_start_us": {"max": max(cta_start), "median": med(cta_start)},
        "rows_per_cta": {"max": max(cta_rows), "median": med(cta_rows), "min": min(cta_rows)},
        "frags_per_cta": {"max": max(cta_frags), "median": med(cta_frags), "min": min(cta_frags)},
        "bins_per_cta": {"max": max(cta_bins), "median": med(cta_bins), "min": min(cta_bins)},
        "slowest_ctas": [{"cta": c, "us": cta_time[c], "rows": cta_rows[c], "frags": cta_frags[c], "bins": cta_bins[c]} for c in order[-4:]],
        "fastest_ctas": [{"cta": c, "us": cta_time[c], "rows": cta_rows[c], "frags": cta_frags[c], "bins": cta_bins[c]} for c in order[:4]],
        "producer_share_blocked_on_empty": mean(prod_wait),
        "consumer_share": {"blocked_pass_through": mean(cons_pass), "blocked_fragment_rows": mean(cons_frag),
                           "bin_loop_with_stores": mean(cons_comp),
                           "other": 1.0 - mean(cons_pass) - mean(cons_frag) - mean(cons_comp)},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=60)
    ap.add_argument("--sets", type=int, default=6)
    ap.add_argument("--src", default=os.path.join(B.CSRC, "roi_align_stream.cu"))
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    ap.add_argument("--keep", default=None, help="write the patched source and the library here instead of a temporary directory")
    args = ap.parse_args()
    import torch
    from detectron.pytorch_b200 import synthetic as S
    if not torch.cuda.is_available():
        raise SystemExit("stream_probe.py: no CUDA device")
    tmp = None
    if args.keep:
        os.makedirs(args.keep, exist_ok=True)
        workdir = args.keep
    else:
        tmp = tempfile.TemporaryDirectory()
        workdir = tmp.name
    so, ptxas = build_probe(args.src, workdir)
    lib = ctypes.CDLL(so)
    lib.probe_forward.restype = ctypes.c_int
    lib.probe_forward.argtypes = [ctypes.c_void_p, ctypes.c_float] + [ctypes.c_int] * 8 + [ctypes.c_void_p] * 3 + [ctypes.c_size_t,
                                                                                                                ctypes.c_void_p]
    lib.probe_ws_bytes.restype = ctypes.c_size_t
    lib.probe_ws_bytes.argtypes = [ctypes.c_int] * 7
    lib.probe_set.restype = ctypes.c_int
    lib.probe_set.argtypes = [ctypes.c_void_p]

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    ctas = torch.cuda.get_device_properties(device).multi_processor_count
    cfg = S.CFG2
    shape, P, scale, sr, R = cfg["shape"], cfg["pooled"], cfg["scale"], cfg["sampling_ratio"], cfg["rois"]
    N, C, H, W = shape
    nsets = max(2, args.sets)
    gen = torch.Generator(device=device); gen.manual_seed(1234)
    feats = [torch.randn(shape, generator=gen, device=device) for _ in range(nsets)]
    rois = [torch.from_numpy(S.make_rois(R, shape, scale, seed=i)).to(device) for i in range(nsets)]
    outs = [torch.empty((R, C, P, P), device=device) for _ in range(nsets)]
    ws_bytes = int(lib.probe_ws_bytes(N, R, H, W, P, P, sr))
    if ws_bytes == 0:
        raise SystemExit("stream_probe.py: the stream path declines cfg2")
    wss = [torch.empty((ws_bytes,), dtype=torch.uint8, device=device) for _ in range(nsets)]
    rec = torch.zeros((ctas, WARPS, NREC), dtype=torch.int64, device=device)
    if lib.probe_set(rec.data_ptr()) != 0:
        raise SystemExit("stream_probe.py: cannot set the record buffer")

    def fwd(i):
        j = i % nsets
        rc = lib.probe_forward(feats[j].data_ptr(), scale, N, R, H, W, C, P, P, sr, rois[j].data_ptr(), outs[j].data_ptr(),
                               wss[j].data_ptr(), ws_bytes, torch.cuda.current_stream().cuda_stream)
        if rc != 0:
            raise RuntimeError("probe_forward failed (status %d)" % rc)

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
    rec_host = rec.cpu().tolist()
    if any(int(rec_host[c][w][11]) != 1 for c in range(ctas) for w in range(WARPS)):
        raise SystemExit("stream_probe.py: some warp wrote no record")
    # the probed source must compute what the library computes (its default path at cfg2)
    from detectron.pytorch_b200 import _lib
    lib_ops = _lib.load()
    fwd(0)
    ref = torch.empty_like(outs[0])
    lws = int(lib_ops.b200_roi_align_workspace_bytes(N, R, H, W, P, P, sr))
    lwsb = torch.empty((max(lws, 1),), dtype=torch.uint8, device=device)
    _lib.check(lib_ops.b200_roi_align_forward_ws(feats[0].data_ptr(), scale, N, R, H, W, C, P, P, sr, rois[0].data_ptr(), ref.data_ptr(),
                                                 lwsb.data_ptr(), lws, torch.cuda.current_stream().cuda_stream), "library forward")
    torch.cuda.synchronize()
    same = bool(torch.equal(outs[0], ref))
    result = {
        "card": card_info(),
        "source": os.path.relpath(os.path.abspath(args.src), ROOT),
        "workload": "RoIAlign forward 1x256x200x272 fp32, 512 RoIs, 7x7, sr=2; CUDA graph of %d calls, %d rotating sets; records of the last call"
                    % (args.calls, nsets),
        "graph_us_per_call": e0.elapsed_time(e1) * 1e3 / args.calls,
        "output_equals_library": same,
        "main_kernel": summarize(rec_host, ctas),
        "ptxas": [l.strip() for l in ptxas.splitlines() if "roi_align_stream_fwd" in l or "spill" in l][:24],
    }
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")
    if tmp is not None:
        tmp.cleanup()
    return 0


if __name__ == "__main__":
    sys.exit(main())
