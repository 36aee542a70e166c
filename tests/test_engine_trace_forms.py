"""CPU test (no GPU needed): the launch sequences of the linear and 1x1 EMASC forms and of the inversion adapter with L > 1 encoder layers
(csrc/engine.cu emasc_forward / adapter_forward, forms derived from the weight table) equal the Python sequencing of the same kernels in
ladi_vton_b200/{vae,adapter}.py, op by op and operand by operand.  Same method as tests/test_engine_trace.py, with the same trace formatter
and data-flow normalisation (tests/kernel_check.py), which also format the full-sequence attention of the extra adapter layers."""
import pytest
import torch

from kernel_check import compare, record  # noqa: F401  (record: a fixture)


def _emasc(ein, eout, seed, **kw):
    from ladi_vton_b200 import EMASC, synthetic as S
    em = EMASC(ein, eout, **kw)
    em._sd = S.random_state_dict(em.param_shapes(), seed)
    em.device = torch.device("cpu")
    em._pack()
    return em


@pytest.mark.parametrize("form", [dict(type="linear", padding=1), dict(kernel_size=1, padding=0), dict(kernel_size=3, padding=1)])
def test_emasc_forms_sequence_matches_python(record, form):
    from ladi_vton_b200 import engine as eng, synthetic as S
    ein, eout = S.emasc_channels(S.SMALL_VAE["block_out_channels"])
    em = _emasc(ein, eout, 3, **form)
    W = em.engine_weights()
    assert ("emasc.0.w2" in W) == (form.get("type") != "linear")
    e = eng.Engine(W, plan_only=True, emasc_scales=5, emasc_in=ein, emasc_out=eout, emasc_stride=[1, 1, 2, 4, 8])
    B, H, Wd = 2, 64, 32
    feats = [torch.zeros((B, H // s, Wd // s, c), dtype=torch.bfloat16) for s, c in zip([1, 1, 2, 4, 8], ein)]
    em(feats, None)
    cpp = e.trace(eng.MODULE_EMASC, B, H, Wd)
    n = compare(record.RECORD, cpp, f"EMASC {form}")
    assert n == (5 if form.get("type") == "linear" else 10)
    k = 1 if form.get("kernel_size") == 1 else 3
    assert all(f"conv k={k} s=1 p={k // 2} " in ln for ln in cpp.splitlines())
    ws = e.workspace_bytes(eng.MODULE_EMASC, B, H, Wd)
    assert ws == 0 if form.get("type") == "linear" else ws > 0  # the linear form writes straight into the caller's outputs


def test_emasc_engine_rejects_unknown_kernel_width():
    from ladi_vton_b200 import engine as eng, lib
    W = {"emasc.0.w1": torch.zeros((64, 5 * 64), dtype=torch.bfloat16), "emasc.0.b1": torch.zeros(64)}
    e = eng.Engine(W, plan_only=True, emasc_scales=1, emasc_in=[64], emasc_out=[64], emasc_stride=[1])
    assert lib.load().ladi_workspace_bytes(e.h, eng.MODULE_EMASC, 1, 8, 8) == -1
    assert b"not a 3x3 or 1x1 kernel" in lib.load().ladi_last_error()


@pytest.mark.parametrize("L", [2, 3])
def test_adapter_layers_sequence_matches_python(record, L):
    from ladi_vton_b200 import InversionAdapter, engine as eng, synthetic as S
    ad = InversionAdapter(input_dim=128, hidden_dim=256, output_dim=512, heads=2, mlp_dim=256, num_encoder_layers=L)
    ad._sd = S.random_state_dict(ad.param_shapes(), 4)
    ad.device = torch.device("cpu"); ad._pack()
    e = eng.Engine(eng.flatten(ad.P, "adapter."), plan_only=True, adapter_dim=128, adapter_heads=2, adapter_mlp=256, adapter_hidden=256, adapter_out=512)
    ad(torch.zeros((3, 17, 128)))
    cpp = e.trace(eng.MODULE_ADAPTER, 3, 17, 0)
    n = compare(record.RECORD, cpp, f"inversion adapter, {L} layers")
    assert sum(ln.startswith("attn_small") for ln in cpp.splitlines()) == L - 1
    assert n == 12 + 7 * (L - 1)


def test_adapter_one_layer_trace_unchanged(record):
    """L = 1: no `adapter.enc*` weights, so the trace is the CLS-only sequence the release checkpoints run."""
    from ladi_vton_b200 import InversionAdapter, engine as eng, synthetic as S
    ad = InversionAdapter(input_dim=128, hidden_dim=256, output_dim=512, heads=2, mlp_dim=256, num_encoder_layers=1)
    ad._sd = S.random_state_dict(ad.param_shapes(), 4)
    ad.device = torch.device("cpu"); ad._pack()
    assert not any(k.startswith("enc") for k in ad.P)
    e = eng.Engine(eng.flatten(ad.P, "adapter."), plan_only=True, adapter_dim=128, adapter_heads=2, adapter_mlp=256, adapter_hidden=256, adapter_out=512)
    cpp = e.trace(eng.MODULE_ADAPTER, 3, 17, 0)
    assert "attn_small" not in cpp and cpp.count("cls_attn") == 1 and len(cpp.splitlines()) == 12
