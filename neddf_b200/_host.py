"""Host plumbing shared by the field networks (NeDDF, NeRF, NeuS): the lifecycle of their C kernel handles and the
assembly of parameter gradients from what a training backward leaves in global memory."""
import ctypes as C

import torch

from . import _lib as L


class KernelHandle:
    """One kind of C handle of a network, for the ABI prefix ``<prefix>_create`` / ``_set_weights`` / ``_destroy``:
    created on first use and on a device change, re-packed when a tensor of ``net._param_tensors()`` was replaced or
    updated in place (``(data_ptr, _version)`` key), destroyed on a device change and by ``release``.

    The object itself holds no state: the handle, its device and the key of its last pack are the network's attributes
    ``<kind>_handle``, ``<kind>_handle_device`` and ``<kind>_packed_key`` (kind "" for the forward handle, "_train" for
    the training one)."""

    def __init__(self, prefix: str, kind: str = "") -> None:
        self.prefix = prefix
        self.names = (kind + "_handle", kind + "_handle_device", kind + "_packed_key")

    def reset(self, net) -> None:
        for name in self.names:
            setattr(net, name, None)

    def get(self, net, device: torch.device):
        lib, name = L.lib(), self.prefix[len("neddf_"):]
        h_attr, dev_attr, key_attr = self.names
        if getattr(net, h_attr) is None or getattr(net, dev_attr) != device:
            self.release(net)
            h = C.c_void_p()
            with torch.cuda.device(device):
                cfg = net._config_struct()
                L.check(getattr(lib, self.prefix + "_create")(C.byref(cfg), C.byref(h)), name + "_create")
            setattr(net, h_attr, h)
            setattr(net, dev_attr, device)
        tensors = net._param_tensors()
        key = tuple((p.data_ptr(), p._version) for p in tensors)
        if key != getattr(net, key_attr):
            for p in tensors:
                if p.dtype != torch.float32 or not p.is_contiguous() or p.device != device:
                    raise RuntimeError("neddf_b200: parameters must be contiguous fp32 tensors on the module's device")
            layers = net._ordered_layers()
            n = len(layers)
            ws = (C.c_void_p * n)(*[l.weight.data_ptr() for l in layers])
            bs = (C.c_void_p * n)(*[l.bias.data_ptr() for l in layers])
            extra = [L.ptr(t) for t in tensors[2 * n:]]  # tensors past the layers' (weight, bias): NeuS's variance
            with torch.cuda.device(device):
                L.check(getattr(lib, self.prefix + "_set_weights")(getattr(net, h_attr), ws, bs, n, *extra,
                                                                      L.stream_ptr(device)), name + "_set_weights")
            setattr(net, key_attr, key)
        return getattr(net, h_attr)

    def release(self, net) -> None:
        h = getattr(net, self.names[0], None)
        if h is not None:
            getattr(L.lib(), self.prefix + "_destroy")(h)
        self.reset(net)


class WeightGrad:
    """Weight and bias gradients of a network's layers over ``n`` samples from the layer inputs X and pre-activation
    gradients G its training backward left in global memory: gW = X^T G as tensor-core split-K GEMMs (neddf_wgrad,
    csrc/wgrad.cu) and bias gradients as column sums of the value rows (neddf_colsum_value_rows), written straight into
    the gradient tensors on the current stream, with a workspace cached on the network per device."""

    def __init__(self, net, device: torch.device, n: int) -> None:
        self.lib, self.device, self.n = L.lib(), device, n
        ws = getattr(net, "_wgrad_ws", None)
        if ws is None or ws.device != device:
            ws = torch.empty(int(self.lib.neddf_wgrad_workspace_bytes()) // 4, device=device, dtype=torch.float32)
            net._wgrad_ws = ws
        self.ws, self.stream = ws, L.stream_ptr(device)

    def empty(self, *shape) -> torch.Tensor:
        return torch.empty(*shape, device=self.device, dtype=torch.float32)

    def into(self, out, row0: int, A, lda: int, ka: int, Bm, rows: int) -> None:
        """out[row0 : row0 + ka, :256] = A[:, :ka]^T Bm over ``rows`` rows (Bm: 256 columns), 128 columns of A at a time."""
        for c0 in range(0, ka, 128):
            kk = min(128, ka - c0)
            L.check(self.lib.neddf_wgrad(L.ptr(A), lda, c0, kk, L.ptr(Bm), 256, rows,
                                         C.c_void_p(out.data_ptr() + 4 * (row0 + c0) * out.shape[1]), out.shape[1], 256,
                                         L.ptr(self.ws), self.stream), "wgrad")

    def colsum(self, Gm, stride: int) -> torch.Tensor:
        """Column sums [256] of the ``n`` value rows of Gm, ``stride`` floats apart."""
        out = self.empty(256)
        L.check(self.lib.neddf_colsum_value_rows(L.ptr(Gm), self.n, stride, L.ptr(out), L.ptr(self.ws), self.stream),
                "colsum")
        return out

    def layer(self, parts, Gm, rows: int, stride: int):
        """[X^T G, bias gradient] of a 256-wide layer whose input X is the concatenation of ``parts`` ((A, columns), with
        lda = columns): the first is [sum of columns, 256], i.e. the gradient of a weight stored [in, out]."""
        gW = self.empty(sum(k for _, k in parts), 256)
        row0 = 0
        for A, k in parts:
            self.into(gW, row0, A, k, k, Gm, rows)
            row0 += k
        return [gW, self.colsum(Gm, stride)]
