"""Host emulation of the SIMT kernels (test infrastructure): see emu_cuda.h."""
from __future__ import annotations

import os
import subprocess
from pathlib import Path

HERE = Path(__file__).resolve().parent
REPO = HERE.parent.parent
BUILD = HERE / "_build"
CXX = "/usr/bin/g++" if Path("/usr/bin/g++").is_file() else "g++"
CSRC = REPO / "simplerecon_b200" / "csrc"
# every kernel file (the wgmma one against the functional model in emu_tc.h) plus the C-ABI front end
UNITS = [CSRC / n for n in ("srcv_api.cu", "srcv_prep.cu", "srcv_dot.cu", "srcv_dot_bwd.cu",
                            "srcv_mlp_generic.cu", "srcv_mlp_bwd.cu", "srcv_mlp_tc.cu", "srcv_tsdf.cu", "srcv_producer.cu", "srcv_mvs.cu", "srcv_mvloss.cu")]
SOURCES = [HERE / "emu_driver.cpp", HERE / "emu_cuda.h", HERE / "emu_tc.h", REPO / "include" / "srcv_b200.h", *sorted(CSRC.glob("*"))]


def build(sanitize: str | None = None, force: bool = False) -> Path:
    """g++-compiles the kernel sources with -DSRCV_HOST_EMU into tests/emu/_build/.
    ``sanitize`` = "address" | "thread" builds an instrumented copy (load it in a process
    started with the matching runtime in LD_PRELOAD, see scripts/emu_sanitize.sh)."""
    BUILD.mkdir(exist_ok=True)
    out = BUILD / (f"libsrcv_emu_{sanitize}.so" if sanitize else "libsrcv_emu.so")
    if not force and out.is_file() and all(p.stat().st_mtime <= out.stat().st_mtime for p in SOURCES if p.is_file()):
        return out
    # The emulation builds exactly the sources and switches the nvcc build ships (build.py
    # NVCC_DEFINES); $SRCV_EMU_DEFINES adds experiment switches.
    from simplerecon_b200.build import NVCC_DEFINES
    defines = [*NVCC_DEFINES, *os.environ.get("SRCV_EMU_DEFINES", "").split()]
    flags = ["-std=c++20", "-pthread", "-fPIC", "-ffp-contract=off", "-DSRCV_HOST_EMU=1", *defines, f"-I{HERE}", "-w"]
    flags += ["-O1", "-g", f"-fsanitize={sanitize}"] if sanitize else ["-O2"]
    objs, procs = [], []
    for src in [HERE / "emu_driver.cpp", *UNITS]:          # one translation unit per source, in parallel
        obj = BUILD / f"{src.stem}{'_' + sanitize if sanitize else ''}.o"
        objs.append(obj)
        procs.append((src, subprocess.Popen([CXX, *flags, "-x", "c++", "-c", str(src), "-o", str(obj)],
                                            stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)))
    for src, p in procs:
        _, err = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"host-emulation build of {src.name} failed:\n{err[-4000:]}")
    r = subprocess.run([CXX, "-shared", "-pthread", *([f"-fsanitize={sanitize}"] if sanitize else []),
                        "-o", str(out), *map(str, objs)], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"host-emulation link failed:\n{r.stderr[-4000:]}")
    return out


def lib_path() -> Path:
    """The library the tests load: $SRCV_EMU_LIB (a sanitizer build) or the plain build."""
    p = os.environ.get("SRCV_EMU_LIB")
    return Path(p) if p else build()


# --------------------------------------------------------------------------------------------- #
# ctypes front end over the emulated library: same structs / prototypes as the product binding   #
# --------------------------------------------------------------------------------------------- #
import ctypes as C  # noqa: E402

import torch  # noqa: E402

from simplerecon_b200 import _native as N  # noqa: E402

_lib = None


def load_or_skip():
    """For fixtures: the emulated library, or pytest.skip when it cannot be built / run here
    (no C++20 host compiler, a thread limit).  The `-m gpu` tier does not depend on it."""
    import pytest
    try:
        return load()
    except (RuntimeError, OSError) as e:
        pytest.skip(f"host emulation unavailable: {str(e)[:300]}")


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        lib = C.CDLL(str(lib_path()))
        for name, (res, args) in N.SYMBOLS.items():
            fn = getattr(lib, name)          # the emulated library exports every ABI symbol
            fn.restype, fn.argtypes = res, args
        lib.emu_set_sms.argtypes = [C.c_int]
        lib.emu_set_sms.restype = None
        lib.emu_can_spawn.argtypes = [C.c_int]
        lib.emu_can_spawn.restype = C.c_int
        if not lib.emu_can_spawn(700):
            raise RuntimeError("this environment does not allow 700 concurrent threads (pids / thread limit)")
        _lib = lib
    return _lib


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _check(lib, st):
    if st != 0:
        raise N.SrcvError(st, lib.srcv_last_error().decode() or lib.srcv_status_string(st).decode())


class Call:
    """Marshals one manager-style argument dict (CPU fp32 tensors) into the C structs."""

    def __init__(self, t: dict, D: int, planes: torch.Tensor | None = None, ramp: torch.Tensor | None = None):
        self.t = {k: v.contiguous() for k, v in t.items() if torch.is_tensor(v)}
        src = self.t["src_feats"]
        self.B, self.K, self.Cc, self.H, self.W = src.shape
        self.D = D
        self.shape = N.Shape(self.B, self.K, self.Cc, self.H, self.W, D)
        self.cams = N.Cameras(self.t["src_extrinsics"].data_ptr(), self.t["src_poses"].data_ptr(),
                              self.t["src_Ks"].data_ptr(), self.t["cur_invK"].data_ptr())
        self.pl = N.Planes()
        self.planes_out = None
        if planes is None:                                    # FROM_RANGE, like the managers' default
            self.ramp = (ramp if ramp is not None else torch.linspace(0, 1, D)).contiguous()
            self.planes_out = torch.empty(self.B, D)
            self.mn, self.mx = self.t["min_depth"].reshape(-1), self.t["max_depth"].reshape(-1)
            self.pl.mode = N.PLANES_FROM_RANGE
            self.pl.planes = None
            self.pl.min_depth, self.pl.max_depth = self.mn.data_ptr(), self.mx.data_ptr()
            self.pl.ramp, self.pl.planes_out = self.ramp.data_ptr(), self.planes_out.data_ptr()
        else:
            self.planes = planes.contiguous()
            self.pl.mode = N.PLANES_PER_PIXEL if planes.dim() == 4 else N.PLANES_PER_PLANE
            self.pl.planes = self.planes.data_ptr()
            self.pl.min_depth = self.pl.max_depth = self.pl.ramp = self.pl.planes_out = None

    def workspace(self, nbytes: int) -> torch.Tensor:
        ws = torch.empty(nbytes + 256, dtype=torch.uint8)
        off = (-ws.data_ptr()) % 256
        return ws[off:off + nbytes]


def dot_forward(t, D, planes=None, want_lowest=True):
    lib, c = load(), Call(t, D, planes)
    cost = torch.full((c.B, D, c.H, c.W), float("nan"))
    lowest = torch.full((c.B, c.H, c.W), float("nan")) if want_lowest else None
    n = lib.srcv_dot_workspace_bytes(C.byref(c.shape))
    ws = c.workspace(n)
    _check(lib, lib.srcv_dot_forward_f32(C.byref(c.shape), _p(c.t["cur_feats"]), _p(c.t["src_feats"]), C.byref(c.cams),
                                         C.byref(c.pl), _p(cost), _p(lowest), _p(ws), n, None))
    return cost, lowest, c.planes_out, lib.srcv_last_variant().decode()


def dot_backward(t, D, gcost, planes=None):
    lib, c = load(), Call(t, D, planes)
    gcur = torch.full_like(c.t["cur_feats"], float("nan"))
    gsrc = torch.full_like(c.t["src_feats"], float("nan"))
    n = lib.srcv_dot_backward_workspace_bytes(C.byref(c.shape))
    ws = c.workspace(n)
    g = gcost.contiguous()
    _check(lib, lib.srcv_dot_backward_f32(C.byref(c.shape), _p(c.t["cur_feats"]), _p(c.t["src_feats"]), C.byref(c.cams),
                                          C.byref(c.pl), _p(g), _p(gcur), _p(gsrc), _p(ws), n, None))
    return gcur, gsrc


def warp_features(t, plane, per_pixel):
    lib, c = load(), Call(t, 1, planes=torch.ones(t["src_feats"].shape[0], 1))
    warped = torch.full((c.B, c.K, c.Cc, c.H, c.W), float("nan"))
    depths = torch.full((c.B, c.K, c.H, c.W), float("nan"))
    mask = torch.full((c.B, c.K, c.H, c.W), float("nan"))
    n = lib.srcv_warp_workspace_bytes(C.byref(c.shape))
    ws = c.workspace(n)
    pln = plane.contiguous()
    _check(lib, lib.srcv_warp_features_f32(C.byref(c.shape), _p(c.t["src_feats"]), C.byref(c.cams), _p(pln),
                                           int(per_pixel), _p(warped), _p(depths), _p(mask), _p(ws), n, None))
    return warped, depths, mask


def _weights(wts):
    keep = [w.detach().contiguous() for w in wts]
    return N.MlpWeights(*[w.data_ptr() for w in keep], keep[0].shape[0], keep[2].shape[0]), keep


def mlp_forward(t, D, wts, planes=None, return_mask=True):
    lib, c = load(), Call(t, D, planes)
    w, keep = _weights(wts)
    cost = torch.full((c.B, D, c.H, c.W), float("nan"))
    lowest = torch.full((c.B, c.H, c.W), float("nan"))
    mask = torch.full((c.B, c.H, c.W), 7, dtype=torch.uint8) if return_mask else None
    n = lib.srcv_mlp_workspace_bytes(C.byref(c.shape), C.byref(w))
    ws = c.workspace(n)
    _check(lib, lib.srcv_mlp_forward_f32(C.byref(c.shape), _p(c.t["cur_feats"]), _p(c.t["src_feats"]), C.byref(c.cams),
                                         C.byref(c.pl), C.byref(w), _p(cost), _p(lowest), _p(mask), _p(ws), n, None))
    return cost, lowest, c.planes_out, (mask.bool() if mask is not None else None), lib.srcv_last_variant().decode()


def mlp_backward(t, D, wts, gcost, planes=None):
    lib, c = load(), Call(t, D, planes)
    w, keep = _weights(wts)
    gcur = torch.full_like(c.t["cur_feats"], float("nan"))
    gsrc = torch.full_like(c.t["src_feats"], float("nan"))
    gw = [torch.full_like(k, float("nan")) for k in keep]
    grads = N.MlpGrads(*[g.data_ptr() for g in gw])
    n = lib.srcv_mlp_backward_workspace_bytes(C.byref(c.shape), C.byref(w))
    ws = c.workspace(n)
    g = gcost.contiguous()
    _check(lib, lib.srcv_mlp_backward_f32(C.byref(c.shape), _p(c.t["cur_feats"]), _p(c.t["src_feats"]), C.byref(c.cams),
                                          C.byref(c.pl), C.byref(w), _p(g), _p(gcur), _p(gsrc), C.byref(grads),
                                          _p(ws), n, None))
    return [gcur, gsrc, *gw]
