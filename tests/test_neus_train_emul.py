"""The NeuS variant's training-backward kernel (csrc/neus_train.cu), executed on the CPU, and its references.

The kernel's tile program (neddf_b200/csrc/neus_train_kernel.cuh) is compiled by g++ into
tests/emul/libneus_train_emul.so (a CTA = 256 OS threads, pthread barrier for __syncthreads) and run on the samples and
upstream gradients (d loss / d density, d loss / d colour per sample, captured with tensor hooks) of fixtures recorded
from the REAL reference's autograd (tests/golden/make_neus_train_golden.py).  The parameter gradients are assembled as
neddf_b200/neus.py does - gW = X^T G over all rows, bias = column sums of the value rows, variance = sum of the per-sample
terms - with numpy standing in for neddf_wgrad, and compared with the reference's.  The restatement the GPU tests use
as the fp64 arbiter (tests/neus_train_oracle.py) is held to the same goldens, and the tanhExp second-derivative quirk
of the reference is pinned by its own recorded values."""
import contextlib
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import neddf_oracle as orc
from tests import nerf_neus_configs as ncfg
from tests import neus_train_oracle as nto
from tests.helpers import GOLDEN, assert_parity, nerr

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emul", "neus_train_emul.cpp")
LIB = os.path.join(HERE, "emul", "libneus_train_emul.so")
CUDA_INC = "/usr/local/cuda/include"
FP = C.POINTER(C.c_float)
BUF_NAMES = ("E4", "XS", "GS", "XC0", "FO", "XC", "GC", "GH", "GV")


class TrainCase:
    def __init__(self, name: str):
        z = np.load(os.path.join(GOLDEN, f"case_neus_train_{name}.npz"), allow_pickle=False)
        self.z = {k: z[k] for k in z.files}
        meta = json.loads(str(self.z["cfg"]))
        self.net_cfg, self.render_cfg = meta["net"], meta["render"]
        self.nc = orc.NeusConfig.from_dict(self.net_cfg)
        self.rc = orc.RenderConfig.from_dict(self.render_cfg)
        cal = [float(v) for v in self.z["cam_calib"]]
        self.cam = orc.CameraPose(torch.from_numpy(self.z["cam_R"]), torch.from_numpy(self.z["cam_T"]), *cal)
        self.separate = "weight_seed_coarse" in self.z
        self.kinked = self.nc.activation_type == "ReLU"

    def net_tag(self, tag):
        return tag if self.separate else "fine"

    def state_dict(self, tag):
        """The parameters the fixture was recorded with (torch layout), rebuilt from its seed."""
        return nto.seeded_state_dict(self.nc, int(self.z[f"weight_seed_{self.net_tag(tag)}"]))

    def weights(self, tag):
        """torch layout ([out,in] weights, [out] biases) in the order of neddf_neus_layer_shapes, + variance."""
        sd = self.state_dict(tag)
        names = [n for n, _, _ in orc.neus_layer_shapes(self.nc)]
        ws = [np.ascontiguousarray(sd[n + ".weight"], np.float32) for n in names]
        bs = [np.ascontiguousarray(sd[n + ".bias"], np.float32) for n in names]
        return names, ws, bs, np.asarray(sd["variance"], np.float32).reshape(1)

    def passes(self):
        """The reference's own rays and edge distances of both passes (make_rays may differ from them in the last bit)."""
        return self.t("ray_dir"), self.t("ray_orig"), (("coarse", self.t("dists_coarse")), ("fine", self.t("dists_fine")))

    def t(self, k):
        return torch.from_numpy(self.z[k])


@pytest.fixture(scope="module")
def emul():
    if shutil.which("g++") is None or not os.path.isdir(CUDA_INC):
        pytest.skip("g++ / CUDA headers not available")
    csrc = os.path.join(HERE, "..", "neddf_b200", "csrc")
    deps = [SRC, os.path.join(HERE, "emul", "emul_common.h"), os.path.join(csrc, "neus_train_kernel.cuh"),
            os.path.join(csrc, "neus_kernel.cuh"), os.path.join(csrc, "simt_tile.cuh"), os.path.join(csrc, "samples.cuh"),
            os.path.join(csrc, "common.cuh"), os.path.join(HERE, "..", "include", "neddf_b200.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I" + CUDA_INC, SRC, "-o", LIB],
                       check=True)
    lib = C.CDLL(LIB)
    lib.neus_train_emul.restype = C.c_int
    return lib


def cfg_struct(nc: orc.NeusConfig):
    from neddf_b200 import _lib as L
    c = L.NeusConfig()
    c.embed_pos_rank, c.embed_dir_rank = nc.embed_pos_rank, nc.embed_dir_rank
    c.sdf_layer_count, c.sdf_layer_width = nc.sdf_layer_count, nc.sdf_layer_width
    c.col_layer_count, c.col_layer_width = nc.col_layer_count, nc.col_layer_width
    c.activation_type = L.ACT_IDS[nc.activation_type]
    c.n_skips = len(nc.skips)
    for i, s in enumerate(nc.skips):
        c.skips[i] = s
    return c


def buffer_shapes(nc: orc.NeusConfig, n: int):
    n_e, n_x, Ls, Lc = 6 * nc.embed_pos_rank, 6 + 6 * nc.embed_dir_rank, nc.sdf_layer_count, nc.col_layer_count
    return {"E4": (n, 4, n_e), "XS": (max(Ls - 1, 1), n, 4, 256), "GS": (Ls, n, 4, 256), "XC0": (n, n_x), "FO": (n, 256),
            "XC": (Lc, n, 256), "GC": (Lc, n, 256), "GH": (n, 3), "GV": (n,)}


def _p(a):
    return None if a is None else a.ctypes.data_as(FP)


def _f32(a, shape=None):
    if a is None:
        return None
    a = np.ascontiguousarray(np.asarray(a, np.float32))
    return a.reshape(shape) if shape is not None else a


def run_backward(lib, nc, ws, bs, variance, g_density, g_color, rays=None, samples=None, g_sdf=None, g_normal=None, nblocks=2):
    """The emulated kernel on rays (ray_dir, ray_orig, dists, sampling_type) or explicit samples (pos, dir [n,3]);
    returns its nine buffers, NaN-filled before the call so that an unwritten element shows."""
    if rays is not None:
        rd, ro, di = (_f32(t.numpy()) for t in rays[:3])
        B, S = di.shape
        n = B * S
    else:
        pos, dd = (_f32(t.numpy(), (-1, 3)) for t in samples)
        n = pos.shape[0]
    buf = {k: np.full(s, np.nan, np.float32) for k, s in buffer_shapes(nc, n).items()}
    arrs = [_f32(g_density, (n,)), _f32(g_color, (n, 3)), _f32(g_sdf, (n,) if g_sdf is not None else None),
            _f32(g_normal, (n, 3) if g_normal is not None else None)]
    gd, gc, gs, gn = arrs
    wp = (FP * len(ws))(*[_p(a) for a in ws])
    bp = (FP * len(bs))(*[_p(a) for a in bs])
    bufs = (FP * 9)(*[_p(buf[k]) for k in BUF_NAMES])
    var = _f32(variance, (1,))
    if rays is not None:
        radius = orc.CONE_RAY_RADIUS if rays[3] == "cone" else 0.0
        rc = lib.neus_train_emul(C.byref(cfg_struct(nc)), wp, bp, len(ws), _p(var), None, None, _p(rd), _p(ro), _p(di),
                                 C.c_longlong(B), C.c_int(S), C.c_int({"point": 0, "cone": 1}[rays[3]]), C.c_float(radius),
                                 _p(gs), _p(gd), _p(gc), _p(gn), bufs, C.c_int(nblocks))
    else:
        rc = lib.neus_train_emul(C.byref(cfg_struct(nc)), wp, bp, len(ws), _p(var), _p(pos), _p(dd), None, None, None,
                                 C.c_longlong(n), C.c_int(0), C.c_int(0), C.c_float(0.0), _p(gs), _p(gd), _p(gc), _p(gn), bufs,
                                 C.c_int(nblocks))
    assert rc == 0
    if nc.sdf_layer_count == 1:
        buf["XS"][:] = 0.0  # unused
    for k, v in buf.items():
        assert np.isfinite(v).all(), k
    return buf, gc


def assemble_grads(nc, names, buf, gc):
    """What neddf_b200/neus.py does with neddf_wgrad / neddf_colsum_value_rows, in float64 numpy: {state_dict key:
    gradient in torch's layout}."""
    Ls, Lc = nc.sdf_layer_count, nc.col_layer_count
    b = {k: v.astype(np.float64) for k, v in buf.items()}
    n = b["FO"].shape[0]
    E4 = b["E4"].reshape(4 * n, -1)
    out = {}
    for l in range(Ls):
        XS = b["XS"][l - 1].reshape(4 * n, 256) if l > 0 else None
        inp = E4 if l == 0 else (np.concatenate([XS, E4], 1) if (l - 1) in nc.skips else XS)
        G = b["GS"][l]
        out[f"layers_sdf.{l}.weight"] = (inp.T @ G.reshape(4 * n, 256)).T
        out[f"layers_sdf.{l}.bias"] = G[:, 0, :].sum(0)
    for l in range(Lc):
        inp = np.concatenate([b["XC0"], b["FO"]], 1) if l == 0 else b["XC"][l - 1]
        out[f"layers_col.{l}.weight"] = (inp.T @ b["GC"][l]).T
        out[f"layers_col.{l}.bias"] = b["GC"][l].sum(0)
    out[f"layers_col.{Lc}.weight"] = b["GH"].T @ b["XC"][Lc - 1]
    out[f"layers_col.{Lc}.bias"] = b["GH"].sum(0)
    out["variance"] = b["GV"].sum()
    assert set(out) == {f"{n}.{p}" for n in names for p in ("weight", "bias")} | {"variance"}
    return out


def oracle_grads(c: TrainCase, dtype, forward=nto.neus_train_forward):
    """Parameter gradients of the fixture's two passes (recorded upstream gradients) by autograd through the training
    restatement, torch layout, keyed like the golden."""
    d, o, passes = c.passes()
    grads = {}
    for tag, dists in passes:
        names, ws, bs, var = c.weights(tag)
        P = nto.params_from_torch(ws, bs, names, var, dtype)
        pos, dd, _ = orc.make_samples(c.rc, d, o, dists)  # the fp32 positions the reference evaluated, then `dtype`
        out = forward(P, c.nc, pos.to(dtype), dd.to(dtype))
        ((out["density"] * c.t(f"up_{tag}_density").to(dtype)).sum() + (out["color"] * c.t(f"up_{tag}_color").to(dtype)).sum()).backward()
        net = "network_" + c.net_tag(tag)
        for k, v in P.items():
            g = v.grad.numpy()
            g = g.T if k.endswith(".weight") else g
            grads[net + "." + k] = grads.get(net + "." + k, 0) + g
    return grads


def compare(c: TrainCase, grads, exact=None, tol=1e-4):
    """Every golden gradient against `grads` (the part neus_train_oracle.fixture_sample keeps); ReLU with the kinked
    rule."""
    checked = 0
    for k in [k for k in c.z if k.startswith("grad_")]:
        g, ref = nto.fixture_sample(np.asarray(grads[k[5:]], np.float64)), c.z[k]
        ex = None if exact is None else nto.fixture_sample(np.asarray(exact[k[5:]], np.float64))
        assert g.shape == ref.shape, (k, g.shape, ref.shape)
        if c.kinked:
            assert_parity(g, ref, tol, kinked=True, what=k + " vs the reference")
            if ex is not None:
                assert nerr(g, ex) < 2e-2, (k, "vs fp64", nerr(g, ex))
        else:
            assert nerr(g, ref) < tol, (k, "vs the reference", nerr(g, ref))
            if ex is not None:
                assert nerr(g, ex) < 5e-5, (k, "vs fp64", nerr(g, ex))
        checked += 1
    assert checked == 2 * len(orc.neus_layer_shapes(c.nc)) * (2 if c.separate else 1) + (2 if c.separate else 1)


def test_reference_tanhexp_second_derivative_is_not_the_true_one():
    """The recorded double backward through the REAL reference's tanhExp Function equals ex (1 - tx^2) (0 above 20),
    which is what the kernel uses - and differs from the true second derivative of x tanh(e^x)."""
    z = np.load(os.path.join(GOLDEN, "case_neus_train_tanhexp.npz"))
    x = torch.from_numpy(z["probe_x"])  # fp32, as recorded (1 - tx^2 cancels at x = 2: compare like with like)
    ref = z["probe_d2"]
    assert np.allclose(ref, nto.ref_tanhexp_d2(x).numpy(), rtol=1e-5, atol=1e-7)
    xs = x.clone().requires_grad_(True)
    (d1,) = torch.autograd.grad(nto.RefTanhExp.apply(xs).sum(), xs, create_graph=True)
    (d2,) = torch.autograd.grad(d1.sum(), xs)
    assert np.allclose(d2.numpy(), ref, rtol=1e-5, atol=1e-7)  # the restatement's Function behaves the same way
    x = x.double()
    xt = x.clone().requires_grad_(True)
    (t1,) = torch.autograd.grad((xt * torch.tanh(torch.exp(xt))).sum(), xt, create_graph=True)
    (true2,) = torch.autograd.grad(t1.sum(), xt)
    i0 = int(np.argmin(np.abs(z["probe_x"])))  # x = 0: 0.420 against the true 0.840
    assert abs(ref[i0] - 0.4200) < 1e-3 and abs(float(true2[i0]) - 0.8399) < 1e-3


@pytest.mark.parametrize("name", ["relu", "tanhexp"])
def test_training_oracle_matches_the_reference_gradients(name):
    """The fp64 restatement (reverse-mode normal, as the reference) against the REAL reference's gradients, and its
    forward-mode twin (the kernel's formulation) against it."""
    c = TrainCase(name)
    rev = oracle_grads(c, torch.float64)
    compare(c, rev)
    fwd = oracle_grads(c, torch.float64, nto.neus_train_forward_jac)
    for k, v in rev.items():
        assert nerr(np.asarray(fwd[k]), np.asarray(v)) < 1e-10, k


@pytest.mark.parametrize("name", ["relu", "tanhexp"])
def test_emulated_backward_matches_the_reference_gradients(emul, name):
    c = TrainCase(name)
    d, o, passes = c.passes()
    grads = {}
    for tag, dists in passes:
        names, ws, bs, var = c.weights(tag)
        buf, gc = run_backward(emul, c.nc, ws, bs, var, c.z[f"up_{tag}_density"], c.z[f"up_{tag}_color"],
                               rays=(d, o, dists, c.rc.sampling_type))
        # the forward the kernel recomputed reproduces the reference's field outputs
        Lc = c.nc.col_layer_count
        zh = buf["XC"][Lc - 1].astype(np.float64) @ ws[-1].astype(np.float64).T + bs[-1]
        col = nto.RefTanhExp.apply(torch.from_numpy(zh)).numpy() if not c.kinked else np.maximum(zh, 0)
        assert nerr(col.reshape(dists.shape + (3,)), c.z[f"field_{tag}_color"]) < 5e-5, (tag, "colour from the recomputed forward")
        assert nerr(buf["FO"][:, 0].reshape(dists.shape), c.z[f"field_{tag}_sdf"]) < 5e-5, (tag, "sdf from the recomputed forward")
        net = "network_" + c.net_tag(tag)
        for k, v in assemble_grads(c.nc, names, buf, gc).items():
            grads[net + "." + k] = grads.get(net + "." + k, 0) + v  # a shared network accumulates both passes
    compare(c, grads, oracle_grads(c, torch.float64))


def test_emulated_backward_optional_gradients_and_ragged_tiles(emul):
    """Upstream gradients on sdf and normal, explicit samples, 1 / 63 / 65 samples (ragged tiles and sub-tiles), a
    shallow tanhExp network with a skip after layer 0, against fp64 autograd through the restatement - including the
    per-layer buffers themselves (g_z / g_Jz of every SDF layer, g_z of every colour layer)."""
    nc = orc.NeusConfig(embed_pos_rank=4, embed_dir_rank=2, sdf_layer_count=3, col_layer_count=2, activation_type="tanhExp",
                        init_variance=0.4, skips=[0])
    P0 = orc.neus_init_params(nc, 5)
    names = [n for n, _, _ in orc.neus_layer_shapes(nc)]
    ws = [np.ascontiguousarray(P0[n + ".weight"].t().numpy()) for n in names]
    bs = [np.ascontiguousarray(P0[n + ".bias"].numpy()) for n in names]
    var = np.array([0.4], np.float32)
    g = torch.Generator().manual_seed(9)
    for n in (1, 63, 65):
        pos = (torch.rand(1, n, 3, generator=g) * 2 - 1) * 0.7
        dd = torch.nn.functional.normalize(torch.randn(1, n, 3, generator=g), dim=-1)
        gs, gd, gc, gn = (torch.randn(1, n, generator=g), torch.randn(1, n, generator=g), torch.randn(1, n, 3, generator=g),
                          torch.randn(1, n, 3, generator=g))
        P = nto.params_from_torch(ws, bs, names, var, torch.float64)
        out, t = nto.neus_train_forward_jac(P, nc, pos.double(), dd.double(), keep=True)
        ((out["sdf"] * gs.double()).sum() + (out["density"] * gd.double()).sum() + (out["color"] * gc.double()).sum()
         + (out["normal"] * gn.double()).sum()).backward()
        buf, gcn = run_backward(emul, nc, ws, bs, var, gd.numpy(), gc.numpy(), samples=(pos, dd), g_sdf=gs.numpy(), g_normal=gn.numpy())
        for l in range(nc.sdf_layer_count):
            ref = np.concatenate([t["sdf_z"][l].grad.numpy()[:, None, :], t["sdf_Jz"][l].grad.numpy()], 1)
            assert nerr(buf["GS"][l], ref) < 2e-5, (n, "GS", l, nerr(buf["GS"][l], ref))
        for l in range(nc.col_layer_count):
            assert nerr(buf["GC"][l], t["col_z"][l].grad.numpy()) < 2e-5, (n, "GC", l)
        got = assemble_grads(nc, names, buf, gcn)
        for k, v in got.items():
            ref = P[k].grad.numpy()
            ref = ref.T if k.endswith(".weight") else ref
            assert nerr(v, ref) < 2e-5, (n, k, nerr(v, ref))


@pytest.mark.parametrize("name", ["S1_one_sdf", "S3_deepest"])  # 0.2 s and 6.5 s on the CPU
def test_emulated_backward_at_table_structures(emul, name):
    """Structures of tests/nerf_neus_configs.py: the sdf from the first layer (ReLU: the kinked rule of
    helpers.assert_parity), both trunks 12 deep (tanhExp); 65 samples with upstream gradients on all four outputs,
    against fp64 autograd through the restatement."""
    nc = ncfg.config(name)
    names = [n for n, _, _ in ncfg.layer_shapes(name)]
    sd = ncfg.state_dict(name)
    ws = [np.ascontiguousarray(sd[n + ".weight"].numpy()) for n in names]
    bs = [np.ascontiguousarray(sd[n + ".bias"].numpy()) for n in names]
    var = sd["variance"].numpy().reshape(1)
    pos, dd, _ = ncfg.samples(1, 65, ncfg.SEED[name] + 1)
    g = torch.Generator().manual_seed(ncfg.SEED[name])
    gs, gd, gc, gn = (torch.randn(1, 65, generator=g), torch.randn(1, 65, generator=g), torch.randn(1, 65, 3, generator=g),
                      torch.randn(1, 65, 3, generator=g))
    P = nto.params_from_torch(ws, bs, names, var, torch.float64)
    out = nto.neus_train_forward_jac(P, nc, pos.double(), dd.double())
    ((out["sdf"] * gs.double()).sum() + (out["density"] * gd.double()).sum() + (out["color"] * gc.double()).sum()
     + (out["normal"] * gn.double()).sum()).backward()
    buf, gcn = run_backward(emul, nc, ws, bs, var, gd.numpy(), gc.numpy(), samples=(pos, dd), g_sdf=gs.numpy(), g_normal=gn.numpy())
    for k, v in assemble_grads(nc, names, buf, gcn).items():
        ref = P[k].grad.numpy()
        ref = ref.T if k.endswith(".weight") else ref
        if nc.activation_type == "ReLU" and np.ndim(v) > 0:
            assert_parity(v, ref, 1e-4, kinked=True, what=k)
        else:
            assert nerr(v, ref) < 2e-5, (k, nerr(v, ref))


class _FakeLib:
    """Stands in for libneddf_b200.so under neddf_b200.NeuS's autograd function on a box without a GPU: the training
    kernel is the host emulation, neddf_wgrad / neddf_colsum_value_rows are numpy on the very pointers, strides and tile
    arguments the glue passes."""

    def __init__(self, emul_lib):
        self.emul, self.handles, self.calls = emul_lib, {}, []

    @staticmethod
    def _arr(p, n):
        addr = p.value if hasattr(p, "value") else p
        return np.ctypeslib.as_array(C.cast(addr, FP), shape=(int(n),))

    def neddf_last_error(self):
        return b"fake"

    def neddf_neus_train_create(self, cfg_ref, h_ref):
        cfg = type(cfg_ref._obj)()
        C.memmove(C.byref(cfg), C.byref(cfg_ref._obj), C.sizeof(cfg))
        h_ref._obj.value = 8192 + len(self.handles)
        self.handles[h_ref._obj.value] = {"cfg": cfg}
        return 0

    def neddf_neus_train_destroy(self, h):
        self.handles.pop(h.value, None)

    def neddf_neus_train_set_weights(self, h, ws, bs, n, var, stream):
        self.handles[h.value].update(w=[C.cast(ws[i], FP) for i in range(n)], b=[C.cast(bs[i], FP) for i in range(n)], n=n,
                                     var=C.cast(var.value, FP))
        return 0

    def _backward(self, h, pos, dirs, rd, ro, dists, n, n_edges, stype, radius, ups, bufs):
        st = self.handles[h.value]
        wp, bp = (FP * st["n"])(*st["w"]), (FP * st["n"])(*st["b"])
        cast = [None if b is None else C.cast(b.value, FP) for b in (pos, dirs, rd, ro, dists) + tuple(ups)]
        bp9 = (FP * 9)(*[C.cast(bufs[i], FP) for i in range(9)])
        self.calls.append("train_backward")
        return self.emul.neus_train_emul(C.byref(st["cfg"]), wp, bp, st["n"], st["var"], *cast[:5], C.c_longlong(n), C.c_int(n_edges),
                                         C.c_int(stype), C.c_float(radius), *cast[5:], bp9, C.c_int(2))

    def neddf_neus_train_backward_rays(self, h, rd, ro, dists, n_rays, n_edges, stype, radius, gs, gd, gc, gn, bufs, stream):
        return self._backward(h, None, None, rd, ro, dists, n_rays, n_edges, stype, radius, (gs, gd, gc, gn), bufs)

    def neddf_neus_train_backward(self, h, pos, dirs, n, gs, gd, gc, gn, bufs, stream):
        return self._backward(h, pos, dirs, None, None, None, n, 0, 0, 0.0, (gs, gd, gc, gn), bufs)

    def neddf_wgrad_workspace_bytes(self):
        return 4096

    def neddf_wgrad(self, a, lda, a_col0, ka, b, ldb, rows, out, ld_out, n_cols, ws, stream):
        assert 0 < ka <= 128 and n_cols == 256 and ld_out == 256 and ldb == 256
        A = self._arr(a, rows * lda).reshape(rows, lda).astype(np.float64)
        B = self._arr(b, rows * ldb).reshape(rows, ldb).astype(np.float64)
        O = self._arr(out, (ka - 1) * ld_out + n_cols)
        res = A[:, a_col0:a_col0 + ka].T @ B[:, :n_cols]
        for m in range(ka):
            O[m * ld_out:m * ld_out + n_cols] = res[m]
        self.calls.append("wgrad")
        return 0

    def neddf_colsum_value_rows(self, g, n_samples, stride, out, ws, stream):
        Gm = self._arr(g, (n_samples - 1) * stride + 256)
        self._arr(out, 256)[:] = np.stack([Gm[s * stride:s * stride + 256] for s in range(n_samples)]).astype(np.float64).sum(0)
        self.calls.append("colsum")
        return 0


def test_autograd_glue_with_emulated_kernels(emul, monkeypatch):
    """neddf_b200.NeuS with training_kernels=True, end to end through torch autograd on CPU tensors: the module's own
    _NeusTrainFn (buffer allocation, pointer arithmetic of the 128-column wgrad tiles, transposes, gradient order,
    variance) over a fake library, against the real reference's parameter gradients.  Default: the call is refused."""
    import neddf_b200
    from neddf_b200 import _lib as L
    c = TrainCase("tanhexp")  # one network for both passes: the gradients of the two calls accumulate
    fake = _FakeLib(emul)
    monkeypatch.setattr(L, "lib", lambda: fake)
    monkeypatch.setattr(L, "stream_ptr", lambda device=None: None)
    monkeypatch.setattr(L, "require_cuda_f32", lambda t, name: t.to(torch.float32).contiguous())
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    d, o, passes = c.passes()
    radius = orc.CONE_RAY_RADIUS if c.rc.sampling_type == "cone" else 0.0
    net = neddf_b200.NeuS(**{k: v for k, v in c.net_cfg.items() if k != "_target_"})
    net.load_state_dict({k: torch.from_numpy(v) for k, v in c.state_dict("fine").items()})
    monkeypatch.setattr(net, "_release", lambda: None)
    names, ws, bs, var = c.weights("fine")

    def launch(a, b, cc, stype, rr, with_normal):  # the inference kernel is not under test: forward values from the oracle
        P = nto.params_from_torch(ws, bs, names, var, torch.float32, requires_grad=False)
        pos, dd, _ = orc.make_samples(c.rc, a, b, cc)
        out = orc.neus_forward(P, c.nc, pos, dd)
        return {"sdf": out["sdf"], "density": out["density"], "color": out["color"], "normal": out["gradients"]}

    monkeypatch.setattr(net, "_launch_forward", launch)
    with pytest.raises(NotImplementedError, match="forward-only"):
        net.forward_rays(d, o, c.t("dists_fine"), c.rc.sampling_type, radius)  # the default
    net.training_kernels = True
    loss = 0
    for tag, dists in passes:
        out = net.forward_rays(d, o, dists, c.rc.sampling_type, radius)
        assert all(out[k].requires_grad for k in ("sdf", "density", "color"))
        loss = loss + (out["density"] * c.t(f"up_{tag}_density")).sum() + (out["color"] * c.t(f"up_{tag}_color")).sum()
    loss.backward()
    assert fake.calls.count("train_backward") == 2
    grads = {"network_fine." + k: p.grad.numpy() for k, p in net.named_parameters()}
    compare(c, grads)
    net._train_handle, net._handle = None, None  # fake handles must never reach the real library's destroy


def _san_build(tmp_path, name, flags):
    exe = str(tmp_path / name)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-ffp-contract=off", "-pthread", "-I" + CUDA_INC] + flags +
                       [os.path.join(HERE, "emul", "neus_train_emul_main.cpp"), "-o", exe], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("sanitizer runtime not available: " + r.stderr[-300:])
    return exe


def test_emulated_backward_under_sanitizers(emul, tmp_path):
    """AddressSanitizer + UBSan (exact-size buffers, float4 alignment) and ThreadSanitizer (best effort) on the emulated
    training-backward kernel (the negative controls that show the detectors see this kind of code live in
    tests/test_neus_emul.py: same harness, same GEMM loop)."""
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66", ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([_san_build(tmp_path, "asan", ["-fsanitize=address,undefined", "-fno-sanitize-recover=all"])], capture_output=True,
                       text=True, env=env, timeout=900)
    assert r.returncode == 0 and "runtime error" not in r.stderr and "AddressSanitizer" not in r.stderr, r.stderr[-1500:]
    assert r.stdout.count("rc 0 checksum") == 2
    r = subprocess.run([_san_build(tmp_path, "tsan", ["-fsanitize=thread"])], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0 and "ThreadSanitizer" not in r.stderr, r.stderr[-1500:]
