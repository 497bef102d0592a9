"""CPU-only: the C-ABI library builds for sm_90a, loads, exports every symbol include/*.h declares,
and validates its arguments before touching CUDA (no compute calls here: there is no GPU)."""
import ctypes
import os
import re

import pytest

from detectron.pytorch_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "b200_roi_ops.h")).read()
    return sorted(set(re.findall(r"B200_API[^;(]*?\b(b200_\w+)\s*\(", text)))


def test_library_builds_and_exports_header_symbols():
    path = build.build()
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    declared = _declared_symbols()
    assert len(declared) >= 13
    for name in declared:
        assert hasattr(lib, name), "header declares %s but the library does not export it" % name
    assert sorted(_lib.EXPORTED_SYMBOLS) == declared       # python binding covers exactly the header


_CTYPES_OF = {"int": ctypes.c_int, "float": ctypes.c_float, "double": ctypes.c_double, "size_t": ctypes.c_size_t,
              "long long": ctypes.c_longlong, "unsigned long long": ctypes.c_ulonglong, "b200_stream_t": ctypes.c_void_p}


def _ctype(decl, is_return=False):
    """ctypes class of one C parameter (or return type) of the header: pointers are c_void_p, char strings c_char_p."""
    decl = " ".join(decl.split())
    if "*" in decl:
        return ctypes.c_char_p if re.fullmatch(r"(const )?char ?\*( ?\w+)?", decl) else ctypes.c_void_p
    words = [w for w in decl.split() if w != "const"]
    if is_return and words == ["void"]:
        return None
    if not is_return and len(words) > 1:
        words = words[:-1]                                   # drop the parameter name
    return _CTYPES_OF[" ".join(words)]


def _header_prototypes():
    text = open(os.path.join(ROOT, "include", "b200_roi_ops.h")).read()
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    text = re.sub(r"//[^\n]*", " ", text)
    protos = {}
    for ret, name, params in re.findall(r"B200_API\s+([^;(]*?)\s*\b(b200_\w+)\s*\(([^)]*)\)\s*;", text):
        params = [p for p in params.split(",") if p.strip()]
        if [p.strip() for p in params] == ["void"]:
            params = []
        protos[name] = (_ctype(ret, is_return=True), [_ctype(p) for p in params])
    return protos


def test_ctypes_signatures_match_the_header():
    """Every prototype of include/b200_roi_ops.h has the same return type and the same argument count and types in the ctypes
    table: an argument of the wrong width there would pass the wrong bits without any error."""
    protos = _header_prototypes()
    assert sorted(protos) == _declared_symbols()
    for name, (restype, argtypes) in protos.items():
        lib_restype, lib_argtypes = _lib._SIGNATURES[name]
        assert lib_restype is restype, "%s returns %s in the header, %s in _lib" % (name, restype, lib_restype)
        assert len(lib_argtypes) == len(argtypes), "%s takes %d arguments in the header, %d in _lib" % (name, len(argtypes), len(lib_argtypes))
        for i, (want, got) in enumerate(zip(argtypes, lib_argtypes)):
            assert got is want, "%s argument %d is %s in the header, %s in _lib" % (name, i, want, got)


def test_reference_named_launchers_are_exported():
    """SURVEY 8b: the reference's own launcher names with the reference's argument lists (include/b200_ref_launchers.h),
    so that lib/.../src/*_cuda.c links unchanged.  Two libraries because the two RoIAlign flavours share their names."""
    build.build()
    text = open(os.path.join(ROOT, "include", "b200_ref_launchers.h")).read()
    body = text[text.index("#ifndef B200_REF_LEGACY_ROI_ALIGN"):]
    main_part, legacy_part = body[:body.rindex("#else")], body[body.rindex("#else"):]
    names = lambda t: sorted(set(re.findall(r"B200_REF_API\s+\w+\s+(\w+)\s*\(", t)))
    lib = ctypes.CDLL(build.compat_lib_path("libb200_ref_launchers.so"))
    assert names(main_part) == ["BilinearSamplerBHWD_updateGradInput_cuda_kernel", "BilinearSamplerBHWD_updateOutput_cuda_kernel",
                                "ROIAlignBackwardLaucher", "ROIAlignForwardLaucher", "ROIPoolBackwardLaucher", "ROIPoolForwardLaucher",
                                "nms_cuda_compute"]
    for n in names(main_part):
        assert hasattr(lib, n), n
    leg = ctypes.CDLL(build.compat_lib_path("libb200_ref_launchers_legacy.so"))
    assert names(legacy_part) == ["ROIAlignBackwardLaucher", "ROIAlignForwardLaucher"]
    for n in names(legacy_part):
        assert hasattr(leg, n), n
    # argument errors come back as 0 (the reference's glue treats 0 as failure), before any CUDA call
    lib.ROIAlignForwardLaucher.restype = ctypes.c_int
    assert lib.ROIAlignForwardLaucher(None, ctypes.c_float(0.25), 4, 0, 10, 3, 7, 7, 2, None, None, None) == 0
    # non-dense strides are refused by the RoICrop launchers
    assert lib.BilinearSamplerBHWD_updateOutput_cuda_kernel(3, 7, 7, 2, 3, 10, 10, 1, None, 300, 100, 10, 2, None, 98, 1, 14, 2,
                                                            None, 147, 49, 7, 1, None) == 0


def test_sm90a_cubin_embedded():
    import subprocess
    path = build.build()
    out = subprocess.run(["cuobjdump", "-lelf", path], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout
    assert "sm_90a" in out


def test_argument_validation_without_gpu():
    lib = _lib.load()
    assert lib.b200_roi_ops_abi_version() == 3
    EINVAL = -1
    # negative / zero dimensions and null pointers are rejected before any CUDA call
    assert lib.b200_roi_align_forward(None, 0.25, 1, 4, 0, 10, 3, 7, 7, 2, None, None, None) == EINVAL
    assert lib.b200_roi_align_forward(None, 0.25, 1, 4, 10, 10, 3, 7, 7, 2, None, None, None) == EINVAL
    assert lib.b200_roi_align_backward(None, 0.25, 1, 4, 10, 10, 3, 7, 7, 2, None, None, None) == EINVAL
    assert lib.b200_roi_pool_forward(None, 0.25, 1, 4, 10, 10, 3, -7, 7, None, None, None, None) == EINVAL
    assert lib.b200_roi_crop_forward(None, None, 1, 3, 10, 10, 2, 7, 7, None, None) == EINVAL
    assert lib.b200_nms(None, 10, 5, 0.7, None, None, None, 0, None) == EINVAL
    assert b"invalid argument" in lib.b200_roi_ops_strerror(EINVAL)
    assert lib.b200_roi_ops_strerror(0) == b"success"
    # workspace sizing is pure host arithmetic: n rows x ceil(n/64) 64-bit words
    assert lib.b200_nms_workspace_bytes(6000) == (6000 * 94 + 94 * 64) * 8      # mask words + transposed diagonal words
    assert lib.b200_nms_workspace_bytes(0) > 0
    assert lib.b200_nms_workspace_bytes(64) == (64 + 64) * 8


def test_workspace_sizing_is_host_arithmetic(lib_option):
    lib = _lib.load()
    # forward fast path: per-RoI tables + per-tile work lists; 0 when the parameters are outside the fast path
    w = lib.b200_roi_align_workspace_bytes(1, 512, 200, 272, 7, 7, 2)
    assert w > 512 * (32 + 28 * 16) and w % 256 == 0
    assert lib.b200_roi_align_workspace_bytes(1, 512, 200, 272, 7, 7, 0) == 0          # adaptive sampling -> generic kernel
    assert lib.b200_roi_align_workspace_bytes(1, 512, 200, 272, 40, 40, 2) == 0        # P * sr > 32 per axis
    assert lib.b200_roi_align_workspace_bytes(1, 0, 200, 272, 7, 7, 2) == 0
    # backward, row-stationary gather path: tables + per-row unit lists + a channel-innermost copy of dY
    wb = lib.b200_roi_align_backward_workspace_bytes(1, 512, 256, 200, 272, 7, 7, 2)
    assert 512 * 256 * 49 * 4 < wb < 512 * 256 * 49 * 4 + (4 << 20) and wb % 256 == 0
    lib_option("B200_ROI_ALIGN_BWD_PATH", "nhwc")     # vector-reduction path: one channel-innermost scratch image of dX
    assert lib.b200_roi_align_backward_workspace_bytes(1, 512, 256, 200, 272, 7, 7, 2) == 256 * 200 * 272 * 4
    lib_option("B200_ROI_ALIGN_BWD_PATH", "generic")
    assert lib.b200_roi_align_backward_workspace_bytes(1, 512, 256, 200, 272, 7, 7, 2) == 0
    lib_option("B200_ROI_ALIGN_BWD_PATH", None)
    assert lib.b200_roi_align_backward_workspace_bytes(0, 512, 256, 200, 272, 7, 7, 2) == 0
    assert lib.b200_roi_align_backward_workspace_bytes(1, 512, 252, 200, 272, 7, 7, 2) == 252 * 200 * 272 * 4     # C % 64 != 0 -> NHWC path
    assert lib.b200_roi_align_backward_workspace_bytes(1, 8, 256, 200, 272, 7, 7, 2) == 0      # tiny gather volume -> scalar atomics
    # batched NMS: sum over problems of (mask words + transposed diagonal words), host arithmetic on a host array
    counts = (ctypes.c_int * 3)(6000, 0, 64)
    assert lib.b200_nms_batched_workspace_bytes(ctypes.cast(counts, ctypes.c_void_p), 3) == ((6000 * 94 + 94 * 64) + (64 + 64)) * 8 + 256
    assert lib.b200_nms_batched_workspace_bytes(ctypes.cast(counts, ctypes.c_void_p), 0) == 0
    assert lib.b200_nms_batched(None, ctypes.cast(counts, ctypes.c_void_p), 3, 5, ctypes.c_float(0.7), None, None, None, 0, None) == -1
    # NULL workspace is legal for the _ws entry points (generic kernels run); bad dims are still rejected first
    assert lib.b200_roi_align_forward_ws(None, 0.25, 1, 4, 10, 10, 3, 0, 7, 2, None, None, None, 0, None) == -1
    assert lib.b200_roi_align_backward_ws(None, 0.25, 1, 4, 10, -1, 3, 7, 7, 2, None, None, None, 0, None) == -1


KEPT_SWITCHES = {"B200_ROI_ALIGN_PATH": b"generic", "B200_ROI_ALIGN_BWD_PATH": b"generic"}
# tuning and timing switches of earlier versions (variants the dispatch never chose, probes with undefined output) and the
# forced backward channels-per-lane and NMS scan variants
RETIRED_SWITCHES = ["B200_" + s for s in ("STREAM_STAGE", "STREAM_PHASES", "STRIP_ROWCOST", "STRIP_PDL", "FWD_ZERO", "BWD_TRCH", "FPN_PATH",
                                          "ROI_ALIGN_BWD_CPL", "NMS_SCAN")]


@pytest.mark.parametrize("name", ["NO_SUCH_SWITCH"] + RETIRED_SWITCHES + sorted(KEPT_SWITCHES))
def test_set_option_accepts_only_path_switches(name):
    """b200_roi_ops_set_option knows the two switches that force a path the dispatch otherwise picks by shape; any other
    name, including the retired tuning, timing and variant switches, is B200_ROI_EINVAL."""
    lib = _lib.load()
    if name not in KEPT_SWITCHES:
        assert lib.b200_roi_ops_set_option(name.encode(), b"x") == -1
        return
    try:
        assert lib.b200_roi_ops_set_option(name.encode(), KEPT_SWITCHES[name]) == 0
    finally:
        assert lib.b200_roi_ops_set_option(name.encode(), None) == 0        # back to the default


def test_round2_entry_points_validate_arguments_without_gpu():
    """Top-k, RoI targets, FPN forward: argument errors are reported before any CUDA call; workspace sizing is host arithmetic."""
    lib = _lib.load()
    EINVAL = -1
    assert lib.b200_topk_batched_workspace_bytes(10) == 10 * 3 * 2048 * 4
    assert lib.b200_topk_batched_workspace_bytes(0) == 0 and lib.b200_topk_batched_workspace_bytes(65) == 0
    assert lib.b200_topk_batched(None, None, None, None, 3, None, None, None, 0, None) == EINVAL
    assert lib.b200_bbox_overlaps(None, 5, None, 4, None, None) == EINVAL
    assert lib.b200_bbox_overlaps(None, 0, None, 4, None, None) == 0                       # nothing to do
    assert lib.b200_roi_assign(None, 3, None, None, 0, None, None, None, None) == EINVAL
    assert lib.b200_roi_select(None, 5, ctypes.c_float(0.5), ctypes.c_float(0.5), ctypes.c_float(0.0), None, None, None, None) == EINVAL
    w4 = (ctypes.c_float * 4)(10, 10, 5, 5)
    assert lib.b200_fast_rcnn_targets(None, None, None, None, None, 4, 5, ctypes.cast(w4, ctypes.c_void_p), 81, 0, ctypes.c_float(1.0),
                                      ctypes.c_float(0.0), None, None, None, None, None, None) == EINVAL      # num_fg > num_keep
    # FPN workspace: the whole pyramid of an 800 x 1333 image (P5 is 25 x 42: staged by cp.async, P2..P4 by TMA)
    H = (ctypes.c_int * 4)(200, 100, 50, 25); W = (ctypes.c_int * 4)(336, 168, 84, 42)
    wf = lib.b200_roi_align_fpn_workspace_bytes(4, ctypes.cast(H, ctypes.c_void_p), ctypes.cast(W, ctypes.c_void_p), 2, 1000, 7, 7, 2)
    assert wf > 1000 * 28 * 16 and wf % 256 == 0
    assert lib.b200_roi_align_forward_fpn(7, None, None, None, None, None, 2, 1000, 256, 7, 7, 2, None, None, None, None, 0, None) == EINVAL
    # single-map workspace covers the quad-strip path's tables, CSR records and temporary records
    w = lib.b200_roi_align_workspace_bytes(1, 512, 200, 272, 7, 7, 2)
    assert w >= 512 * 28 * 16 + 512 * 196 * 24


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, "detectron")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, fn)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, re.M), fn
                assert "liboracle" not in text and "oracle/_ref" not in text, fn
