"""What every engine model class (UNet, VAE, EMASC, inversion adapter, CLIP towers, warping modules, metrics networks) shares with the
reference object it replaces: a strict `load_state_dict` against the class's `param_shapes()`, a CUDA-only `.to()` that packs the
weights for the kernels, and the choice between the engine handle (one ABI call into csrc/engine.cu) and the Python sequencing."""
import torch

from . import engine as eng, lib, ops


class _Cfg(dict):
    """A config dict whose keys also read as attributes (`config.block_out_channels`), like the diffusers / transformers configs."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


class PackedModule:
    """Subclasses define `param_shapes()` -> {state-dict key: shape} and `_pack_weights()`, which packs `self._sd` for `self.device`;
    `_make_engine()` builds their engine handle, if they have one."""
    device = torch.device("cpu")  # until moved: packing happens on the first CUDA device the module is moved to
    _sd = None  # the state dict, kept until packed from device-resident tensors
    P = None  # the packed weights
    pack_gen = 0  # bumped by every pack: captured graphs hold the packed weights' addresses (pipeline._graph_key)
    engine = None

    def eval(self):
        return self

    def requires_grad_(self, flag=False):
        return self

    def optional(self, key):
        """A parameter the state dict may leave out."""
        return False

    def ignorable(self, key):
        """A key outside param_shapes() that a strict load accepts and drops."""
        return False

    def load_state_dict(self, sd, strict=True):
        want = self.param_shapes()
        missing = [k for k in want if k not in sd and not self.optional(k)]
        misshaped = [k for k in want if k in sd and tuple(sd[k].shape) != tuple(want[k])]
        unexpected = [k for k in sd if k not in want and not self.ignorable(k)] if strict else []
        if missing or misshaped or unexpected:
            raise RuntimeError(f"{type(self).__name__} state_dict mismatch: missing {missing[:4]}, misshaped {misshaped[:4]}, "
                               f"unexpected {unexpected[:4]}")
        self._sd = {k: v.detach() for k, v in sd.items() if k in want}
        if self.device.type == "cuda":
            self._pack()
        return self

    def to(self, device=None, dtype=None, **kw):
        """Packs the weights for a CUDA device.  A dtype, also in the device's place, is accepted and ignored: the precision is fixed."""
        if device is None or isinstance(device, torch.dtype):
            return self
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError(f"ladi_vton_b200 {type(self).__name__} runs on CUDA (sm_90a) only; there is no CPU path")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if self.pack_gen and device == self.device:
            return self  # already packed here: re-packing would free weights a captured graph still points at
        if self.pack_gen and self._sd is None:
            raise RuntimeError(f"the state dict was released after packing; call load_state_dict again to move the {type(self).__name__}")
        self.device = device
        if self._sd is not None:
            self._pack()
        return self

    def _pack(self):
        self._pack_weights()
        self.pack_gen += 1
        self.engine = None
        if eng.enabled() and self.device.type == "cuda":
            self.engine = self._make_engine()
        if any(v.is_cuda for v in self._sd.values()):
            self._sd = None  # device-resident fp32 sources (3.5 GB for the full UNet) are not kept beside the bf16 pack

    def _make_engine(self):
        return None

    def use_engine(self):
        """True where a call goes to the engine handle.  Profiling (ops.PROFILE) and recording (lib.RECORD) need the Python
        sequencing of the same kernels, which issues them one by one."""
        return self.engine is not None and ops.PROFILE is None and lib.RECORD is None
