"""CPU test (no GPU needed): the launch sequences of the module-level C ABI (csrc/engine.cu: ladi_unet_forward, ladi_vae_encode,
ladi_vae_decode_emasc, ladi_emasc_forward, ladi_inversion_adapter_forward) are pinned, op by op and operand by operand, to the Python
sequencing of the same kernels in ladi_vton_b200/{unet,vae,adapter}.py -- the sequencing every GPU parity test of round 1 validated
against the oracle.  The C++ side is walked in plan mode (no launches; `ladi_engine_trace`), the Python side runs on CPU tensors with
the ABI calls recorded instead of executed (`lib.RECORD`).  Addresses differ (workspace offsets vs torch allocations), so both traces
are normalised to (buffer id, byte offset) by data flow: a buffer is born where an op writes it, reads resolve to the youngest buffer
containing the address, external operands (weights, inputs) are numbered by first appearance (normalise in tests/kernel_check.py)."""
import pytest
import torch

from kernel_check import compare, record  # noqa: F401  (record: a fixture)


def _cpu_pack(model):
    model.device = torch.device("cpu")
    model._pack()
    return model


@pytest.mark.parametrize("B,h,w", [(2, 16, 8), (3, 8, 16)])
@pytest.mark.parametrize("fuse", ["1", "0"])
def test_unet_sequence_matches_python(record, monkeypatch, B, h, w, fuse):
    from ladi_vton_b200 import UNet2DConditionModel, engine as eng, synthetic as S, unet_param_shapes
    monkeypatch.setenv("LADI_UP2X", fuse)
    unet = UNet2DConditionModel(**S.SMALL_UNET)
    unet._sd = S.random_state_dict(unet_param_shapes(S.SMALL_UNET), 1)
    _cpu_pack(unet)
    e = eng.Engine(eng.flatten(unet.P), plan_only=True, **unet.engine_config())
    assert e.query(eng.Q_TEMB_TOTAL) == unet.temb_total and e.query(eng.Q_KV_TOTAL) == unet.kv_total and e.query(eng.Q_IN_PITCH) == unet.in_pitch
    unet._steps = torch.zeros((4, unet.temb_total))
    unet._ctx = torch.zeros((B, 77, unet.kv_total), dtype=torch.bfloat16)
    x = torch.zeros((B, h, w, unet.in_pitch), dtype=torch.bfloat16)
    unet.forward_nhwc(x, torch.zeros(2, dtype=torch.int32))
    n = compare(record.RECORD, e.trace(eng.MODULE_UNET, B, h, w), "UNet forward")
    assert n > 300
    assert e.workspace_bytes(eng.MODULE_UNET, B, h, w) > 0
    # the step-invariant table: sinusoid (device kernel in C++, host trig in the Python sequencing) -> time MLP -> all time_emb_proj: the three GEMMs must match
    record.RECORD.clear()
    unet._steps = unet._steps_key = None
    unet.plan_steps([981, 961, 941])
    cpp = "\n".join(l for l in e.trace(eng.MODULE_UNET_PLAN, 3, 0, 0).splitlines() if not l.startswith("timestep_embedding"))
    assert compare(record.RECORD, cpp, "UNet plan_steps") == 3


@pytest.mark.parametrize("fuse", ["1", "0"])
def test_vae_emasc_sequences_match_python(record, monkeypatch, fuse):
    from ladi_vton_b200 import AutoencoderKL, EMASC, engine as eng, synthetic as S
    from ladi_vton_b200.vae import vae_param_shapes
    monkeypatch.setenv("LADI_UP2X", fuse)
    vae = AutoencoderKL(**S.SMALL_VAE)
    vae._sd = S.random_state_dict(vae_param_shapes(S.SMALL_VAE), 2)
    _cpu_pack(vae)
    e = eng.Engine(eng.flatten(vae.P), plan_only=True, **vae.engine_config())
    B, H, W = 2, 64, 32
    x = torch.zeros((B, H, W, 8), dtype=torch.bfloat16)
    mom, feats = vae.encode_nhwc(x, nhwc=True)
    compare(record.RECORD, e.trace(eng.MODULE_VAE_ENCODE, B, H, W), "VAE encode")
    # EMASC on the retained features (hubconf.py:41-42 channel plan), then decode with the skips
    ein, eout = S.emasc_channels(S.SMALL_VAE["block_out_channels"])
    em = EMASC(ein, eout)
    em._sd = S.random_state_dict(S.emasc_param_shapes(ein, eout), 3)
    em.device = torch.device("cpu"); em._pack()
    W_ = {}
    for i, (w1, b1, w2, b2) in enumerate(em.P):
        W_.update({f"emasc.{i}.w1": w1, f"emasc.{i}.b1": b1, f"emasc.{i}.w2": w2, f"emasc.{i}.b2": b2})
    ee = eng.Engine(W_, plan_only=True, emasc_scales=5, emasc_in=ein, emasc_out=eout, emasc_stride=[1, 1, 2, 4, 8])
    record.RECORD.clear()
    sel = [feats[i] if i != 2 else feats[i].clone() for i in range(1, 6)]  # (features 1 and 2 are one tensor; the plan walk uses five distinct operands)
    inter = em(sel, None)
    compare(record.RECORD, ee.trace(eng.MODULE_EMASC, B, H, W), "EMASC")
    record.RECORD.clear()
    z = torch.zeros((B, 4, H // 8, W // 8))
    vae.decode_nhwc(z, inter, [1, 2, 3, 4, 5])
    recs = [r for r in record.RECORD if r[0] != "ladi_nchw_f32_to_nhwc_bf16"]  # the latent layout kernel stays on the Python side of the ABI
    compare(recs, e.trace(eng.MODULE_VAE_DECODE, B, H // 8, W // 8), "VAE decode")


def test_adapter_sequence_matches_python(record):
    from ladi_vton_b200 import InversionAdapter, engine as eng, synthetic as S
    ad = InversionAdapter(input_dim=128, hidden_dim=256, output_dim=512, heads=2, mlp_dim=256)
    ad._sd = S.random_state_dict(ad.param_shapes(), 4)
    ad.device = torch.device("cpu"); ad._pack()
    e = eng.Engine(eng.flatten(ad.P, "adapter."), plan_only=True, adapter_dim=128, adapter_heads=2, adapter_mlp=256, adapter_hidden=256, adapter_out=512)
    ad(torch.zeros((3, 17, 128)))
    compare(record.RECORD, e.trace(eng.MODULE_ADAPTER, 3, 17, 0), "inversion adapter")


def test_engine_errors_and_workspace_monotone():
    from ladi_vton_b200 import engine as eng, lib
    e = eng.Engine({}, plan_only=True, unet_channels=[64, 128, 256, 256], unet_heads=[1, 2, 4, 4], unet_down_attn=[1, 1, 1, 0], unet_up_attn=[0, 1, 1, 1],
                   unet_layers_per_block=2, unet_in_channels=31, unet_out_channels=4, unet_norm_eps=1e-5, norm_groups=32, fuse_upsample=1)
    assert lib.load().ladi_workspace_bytes(e.h, eng.MODULE_UNET, 2, 16, 8) == -1  # no weights in the table
    assert b"not in the table" in lib.load().ladi_last_error()
    assert lib.load().ladi_workspace_bytes(e.h, 99, 1, 8, 8) == -1
    assert lib.load().ladi_unet_forward(None, None, None, None, None, 1, 1, 1, 1, None, None, 0, None) != 0
