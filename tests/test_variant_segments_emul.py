"""The segment view of the NeRF and NeuS forward kernels (early ray termination), executed on the CPU.

The tile programs of csrc/nerf_simt.cu and csrc/neus_simt.cu (nerf_kernel.cuh, neus_kernel.cuh) are compiled by g++
into host emulations (tests/emul/nerf_emul.cpp, neus_segment_emul.cpp; a CTA = 256 OS threads, pthread barrier for
__syncthreads).  On a golden's weights and rays, depth segments over a ray list that skips rays must reproduce the
whole-row launch bit for bit on the entries they evaluate and leave every other entry alone: each sample's arithmetic
does not depend on which samples share its tile.  The sanitizer run covers the segment path of both kernels."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import neddf_oracle as orc
from tests.test_nerf_oracle import NerfCase
from tests.test_nerf_train_emul import cfg_struct as nerf_cfg_struct
from tests.test_nerf_train_emul import torch_layout_weights
from tests.test_neus_emul import _cfg_struct as neus_cfg_struct
from tests.test_neus_oracle import NeusCase

HERE = os.path.dirname(os.path.abspath(__file__))
EMUL = os.path.join(HERE, "emul")
CSRC = os.path.join(HERE, "..", "neddf_b200", "csrc")
CUDA_INC = "/usr/local/cuda/include"
FP = C.POINTER(C.c_float)
I32P = C.POINTER(C.c_int32)
SENTINEL = np.float32(-7.25)  # what the caller's arrays hold where no launch may write
RAY_LIST = [3, 0, 2]          # of 4 rays: ray 1 is not listed, the order carries no meaning


def _build(src: str, lib: str, headers):
    deps = [os.path.join(EMUL, src), os.path.join(EMUL, "emul_common.h"), os.path.join(HERE, "..", "include", "neddf_b200.h")] + \
        [os.path.join(CSRC, h) for h in headers]
    out = os.path.join(EMUL, lib)
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I" + CUDA_INC,
                        os.path.join(EMUL, src), "-o", out], check=True)
    return C.CDLL(out)


@pytest.fixture(scope="module")
def libs():
    if shutil.which("g++") is None or not os.path.isdir(CUDA_INC):
        pytest.skip("g++ / CUDA headers not available")
    common = ["simt_tile.cuh", "common.cuh"]
    nerf = _build("nerf_emul.cpp", "libnerf_emul.so", ["nerf_kernel.cuh", "field_math.cuh"] + common)
    neus = _build("neus_segment_emul.cpp", "libneus_segment_emul.so", ["neus_kernel.cuh"] + common)
    for f in (nerf.nerf_emul_forward_segment, neus.neus_emul_forward_segment):
        f.restype = C.c_int
    return nerf, neus


def _p(a, t=FP):
    return None if a is None else a.ctypes.data_as(t)


def _f32(t):
    return np.ascontiguousarray(t.numpy(), np.float32)


def _segments(E: int, K: int):
    """The renderer's depth segments (NeRFRender._fine_pass_terminated): bounds round(k E / K)."""
    b = [round(k * E / K) for k in range(K + 1)]
    return [(b[k], b[k + 1] - b[k]) for k in range(K)]


def _check_segments(launch, n_rays: int, E: int):
    """launch(density, color, edge0, seg_len, ray_index, n_active): whole rows for seg_len = 0.  Segment launches over 2, 3
    and E segments into sentinel-filled arrays: after every launch the listed rays' entries up to the segment's end are
    the whole-row launch's bit for bit, everything else still holds the sentinel."""
    den = np.full((n_rays, E), np.nan, np.float32)
    col = np.full((n_rays, E, 3), np.nan, np.float32)
    assert launch(den, col, 0, 0, None, None) == 0
    assert np.isfinite(den).all() and np.isfinite(col).all()
    idx = np.array(RAY_LIST, np.int32)
    n_active = np.array([len(idx)], np.int32)
    listed = np.zeros(n_rays, bool)
    listed[idx] = True
    for K in (2, 3, E):
        sden = np.full((n_rays, E), SENTINEL, np.float32)
        scol = np.full((n_rays, E, 3), SENTINEL, np.float32)
        for e0, seg in _segments(E, K):
            assert launch(sden, scol, e0, seg, idx, n_active) == 0
            done = listed[:, None] & (np.arange(E)[None, :] < e0 + seg)
            assert np.array_equal(sden[done].view(np.uint32), den[done].view(np.uint32)), (K, e0)
            assert np.array_equal(scol[done].view(np.uint32), col[done].view(np.uint32)), (K, e0)
            assert (sden[~done] == SENTINEL).all() and (scol[~done] == SENTINEL).all(), (K, e0)


@pytest.mark.parametrize("name", ["relu", "tanhexp"])
def test_emulated_nerf_segments_equal_whole_rows(libs, name):
    """NeRF goldens (ReLU: shared network, cone sampling; tanhExp: separate networks, point sampling), four golden rays
    at the first 24 edges of the coarse pass."""
    lib = libs[0]
    c = NerfCase(name)
    d, o = orc.make_rays(c.t("uv"), c.cam)
    dists = orc.coarse_dists(c.rc, c.t("u_coarse"))[:4, :24]
    rd, ro, di = _f32(d[:4]), _f32(o[:4]), _f32(dists)
    ws, bs = torch_layout_weights(c, "coarse")
    wp, bp = (FP * len(ws))(*[_p(a) for a in ws]), (FP * len(bs))(*[_p(a) for a in bs])
    lowpass = orc.lowpass_scale(c.nc.embed_pos_rank, c.alpha).numpy().astype(np.float32)
    cfg = nerf_cfg_struct(c.nc)
    radius = orc.CONE_RAY_RADIUS if c.rc.sampling_type == "cone" else 0.0
    n_rays, E = di.shape

    def launch(den, col, e0, seg, idx, n_active):
        return lib.nerf_emul_forward_segment(C.byref(cfg), wp, bp, len(ws), _p(lowpass), _p(rd), _p(ro), _p(di), C.c_longlong(n_rays),
                                             C.c_int(E), C.c_int({"point": 0, "cone": 1}[c.rc.sampling_type]), C.c_float(radius),
                                             C.c_int(e0), C.c_int(seg), _p(idx, I32P), _p(n_active, I32P), _p(den), _p(col), C.c_int(2))

    _check_segments(launch, n_rays, E)


@pytest.mark.parametrize("name", ["relu", "tanhexp"])
def test_emulated_neus_segments_equal_whole_rows(libs, name):
    """NeuS goldens (ReLU 8 + 8 layers, cone sampling; tanhExp 6 + 3, point sampling), four golden rays at the first
    24 edges of the coarse pass."""
    lib = libs[1]
    c = NeusCase(name)
    d, o = orc.make_rays(c.t("uv"), c.cam)
    dists = orc.coarse_dists(c.rc, c.t("u_coarse"))[:4, :24]
    rd, ro, di = _f32(d[:4]), _f32(o[:4]), _f32(dists)
    pre = "w_coarse." if "w_coarse.layers_sdf.0.weight" in c.z else "w_fine."
    names = [n for n, _, _ in orc.neus_layer_shapes(c.nc)]
    ws = [np.ascontiguousarray(c.z[pre + n + ".weight"], np.float32) for n in names]
    bs = [np.ascontiguousarray(c.z[pre + n + ".bias"], np.float32) for n in names]
    var = np.ascontiguousarray(c.z[pre + "variance"], np.float32).reshape(1)
    wp, bp = (FP * len(ws))(*[_p(a) for a in ws]), (FP * len(bs))(*[_p(a) for a in bs])
    cfg = neus_cfg_struct(c.nc)
    stype = C.c_int({"point": 0, "cone": 1}[c.rc.sampling_type])
    radius = C.c_float(orc.CONE_RAY_RADIUS if c.rc.sampling_type == "cone" else 0.0)
    n_rays, E = di.shape

    def launch(den, col, e0, seg, idx, n_active):
        return lib.neus_emul_forward_segment(C.byref(cfg), wp, bp, len(ws), _p(var), _p(rd), _p(ro), _p(di), C.c_longlong(n_rays), C.c_int(E),
                                             stype, radius, C.c_int(e0), C.c_int(seg), _p(idx, I32P), _p(n_active, I32P), _p(den), _p(col),
                                             C.c_int(2))

    _check_segments(launch, n_rays, E)


def _san_build(tmp_path, name, flags):
    exe = str(tmp_path / name)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-ffp-contract=off", "-pthread", "-I" + CUDA_INC] + flags +
                       [os.path.join(EMUL, "segment_emul_main.cpp"), "-o", exe], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("sanitizer runtime not available: " + r.stderr[-300:])
    return exe


def test_emulated_segments_under_sanitizers(libs, tmp_path):
    """AddressSanitizer + UBSan (memcheck: exact-size [n_rays, n_edges] outputs, the ray list, float4 alignment) and
    ThreadSanitizer (racecheck, best effort) on a whole-row launch and a segment launch of both kernels over a ray list
    that skips rays, two tiles over two CTAs (the negative controls that show the detectors see this code live in
    tests/test_neus_emul.py: same harness, same tile skeleton)."""
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66", ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([_san_build(tmp_path, "asan", ["-fsanitize=address,undefined", "-fno-sanitize-recover=all"])], capture_output=True,
                       text=True, env=env, timeout=600)
    assert r.returncode == 0 and "runtime error" not in r.stderr and "AddressSanitizer" not in r.stderr, r.stderr[-1500:]
    assert r.stdout.count("segment rc 0 mismatches 0") == 2, r.stdout
    r = subprocess.run([_san_build(tmp_path, "tsan", ["-fsanitize=thread"])], capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0 and "ThreadSanitizer" not in r.stderr, r.stderr[-1500:]
