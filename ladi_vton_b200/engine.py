"""ctypes side of the module-level C ABI (include/ladi_b200.h, csrc/engine.cu): an opaque engine handle built from a module's packed
weights, and the per-module entry points -- `ladi_unet_forward`, `ladi_vae_encode`, `ladi_vae_decode_emasc`, `ladi_emasc_forward`,
`ladi_inversion_adapter_forward`, `ladi_denoise_loop` -- the launch sequences of which live in C++.  The Python model classes
(unet.py / vae.py / adapter.py) are thin callers of these; their own Python sequencing of the same kernels is kept for two purposes only:
per-launch instrumentation (ops.PROFILE, bench.py's roofline pass) and the CPU test that pins the C++ sequence to it op by op
(tests/test_engine_trace.py).  Env LADI_ENGINE=0 forces the Python sequencing (A/B).  When a model builds its handle and when a call
takes it is decided in one place, module.PackedModule (`_pack`, `use_engine`).
"""
import ctypes as C
import os

import torch

from . import lib

MODULE_UNET, MODULE_VAE_ENCODE, MODULE_VAE_DECODE, MODULE_EMASC, MODULE_ADAPTER, MODULE_UNET_PLAN = 0, 1, 2, 3, 4, 5
Q_TEMB_TOTAL, Q_KV_TOTAL, Q_IN_PITCH = 0, 1, 2


def enabled():
    return os.environ.get("LADI_ENGINE", "1") != "0"


def flatten(P, prefix=""):
    """Packed-weight dict (tensors, or tuples of tensors such as (gamma, beta)) -> {name: tensor}; tuple entries become name.0, name.1."""
    out = {}
    for k, v in P.items():
        if isinstance(v, (tuple, list)):
            for i, t in enumerate(v):
                out[f"{prefix}{k}.{i}"] = t
        else:
            out[prefix + k] = v
    return out


class Engine:
    def __init__(self, weights, plan_only=False, **cfg):
        """weights: {name: tensor} (device tensors; any tensors when plan_only); cfg: fields of ladi_engine_config (lists for the arrays)."""
        l = lib.load()
        c = lib.EngineConfig()
        for k, v in cfg.items():
            if isinstance(v, (list, tuple)):
                arr = getattr(c, k)
                for i, x in enumerate(v):
                    arr[i] = int(x)
            else:
                setattr(c, k, v)
        c.plan_only = int(plan_only)
        self._keep = dict(weights)  # the handle stores raw pointers: keep the tensors alive as long as it lives
        names = [n.encode() for n in self._keep]
        table = (lib.Weight * max(1, len(names)))()
        for i, (n, t) in enumerate(self._keep.items()):
            table[i].name = names[i]
            table[i].ptr = t.data_ptr()
            table[i].rows = int(t.shape[0]) if t.dim() == 2 else 1
            table[i].cols = int(t.shape[1]) if t.dim() == 2 else int(t.numel())
        self._names = names
        h = C.c_void_p()
        rc = l.ladi_engine_create(C.byref(c), table, len(names), C.byref(h))
        if rc != 0:
            raise RuntimeError(f"ladi_engine_create failed ({rc}): {l.ladi_last_error().decode()}")
        self.h, self.cfg, self._ws = h, c, {}
        self.device = next(iter(self._keep.values())).device if self._keep else torch.device("cpu")

    def __del__(self):
        try:
            if getattr(self, "h", None):
                lib.load().ladi_engine_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def query(self, what):
        return lib.load().ladi_engine_query(self.h, what)

    def workspace_bytes(self, module, batch, height, width):
        n = lib.load().ladi_workspace_bytes(self.h, module, batch, height, width)
        if n < 0:
            raise RuntimeError(f"ladi_workspace_bytes failed: {lib.load().ladi_last_error().decode()}")
        return n

    def trace(self, module, batch, height, width):
        """The launch sequence (one op per line) of one call of `module` at this shape, from a plan-mode walk of the C++ body."""
        self.workspace_bytes(module, batch, height, width)
        return lib.load().ladi_engine_trace(self.h).decode()

    def workspace(self, module, batch, height, width):
        """Caller-owned activation workspace for (module, shape): allocated once and kept (captured graphs hold its address)."""
        key = (module, batch, height, width)
        ws = self._ws.get(key)
        if ws is None:
            ws = self._ws[key] = torch.empty(max(256, self.workspace_bytes(module, batch, height, width)), dtype=torch.uint8, device=self.device)
        return ws


def ptr_array(tensors, n=None):
    """-> (void* [n]) of data pointers (None -> NULL)."""
    n = len(tensors) if n is None else n
    arr = (C.c_void_p * n)()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr() if t is not None else None
    return arr
