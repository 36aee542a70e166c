"""ORACLE (test infrastructure only) -- the EMASC forms src/eval.py and train_emasc.py build besides the hub's nonlinear 3x3
(parts.EMASC): fp32 CPU restatement of src/models/emasc.py:11-40 for
  * type 'linear': one Conv2d per scale, always 3x3 (the reference ignores `kernel_size`, emasc.py:21-24); keys conv.{i}.{weight,bias};
  * type 'nonlinear' with any kernel_size / padding: Conv(k) -> SiLU -> Conv(k); keys conv.{i}.{0,2}.{weight,bias}.
Pinned bit for bit against the reference class (tests/golden/emasc_forms.npz, tests/golden/make_forms_golden.py).

Only tests/ may import this module.
"""
import torch.nn as nn


class EMASC(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size=3, padding=1, type="nonlinear"):
        super().__init__()
        if type == "linear":
            self.conv = nn.ModuleList([nn.Conv2d(ci, co, 3, padding=padding) for ci, co in zip(in_channels, out_channels)])
            return
        k, p = kernel_size, padding
        self.conv = nn.ModuleList([
            nn.Sequential(nn.Conv2d(ci, ci, k, padding=p), nn.SiLU(), nn.Conv2d(ci, co, k, padding=p))
            for ci, co in zip(in_channels, out_channels)])

    def forward(self, feats):
        return [m(f) for m, f in zip(self.conv, feats)]
