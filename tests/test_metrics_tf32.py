"""Host-side tests of the metric networks' tf32 precision (metrics.py precision="tf32", val_metrics.py --precision): the fp32 weight packing
(BatchNorm fold in float64, (ky, kx, c) im2col columns, K padded with zeros to a multiple of 4) against F.conv2d in float64 for every kernel
shape of the two networks, the CLI flag and the statistics-cache name, and a census of the ABI calls the tf32 networks record
(`lib.RECORD`): every GEMM is a `ladi_gemm_tf32` whose operands and output slice obey the kernel's placement rules, and no bf16 kernel runs.
No GPU needed."""
import pytest
import torch
import torch.nn.functional as F

from kernel_check import cpu_pack, recorded


def _im2col_rows(x_nchw, kernel, stride, padding, k_pad):
    (kh, kw), (sh, sw), (ph, pw) = kernel, stride, padding
    xp = F.pad(x_nchw, (pw, pw, ph, ph))
    n, c = x_nchw.shape[:2]
    oh, ow = (xp.shape[2] - kh) // sh + 1, (xp.shape[3] - kw) // sw + 1
    cols = [xp[:, :, ky:ky + sh * (oh - 1) + 1:sh, kx:kx + sw * (ow - 1) + 1:sw] for ky in range(kh) for kx in range(kw)]
    rows = torch.stack(cols, 1).permute(0, 3, 4, 1, 2).reshape(n * oh * ow, kh * kw * c)
    return F.pad(rows, (0, k_pad - rows.shape[1])), (n, oh, ow)


# every kernel shape of the FID Inception-v3 and the LPIPS AlexNet (c_in small but with the networks' remainders mod 4)
SHAPES = [("1x1", (1, 1), (1, 1), (0, 0), 20), ("3x3 valid", (3, 3), (1, 1), (0, 0), 32), ("3x3 same", (3, 3), (1, 1), (1, 1), 24),
          ("3x3 stride 2", (3, 3), (2, 2), (0, 0), 16), ("5x5", (5, 5), (1, 1), (2, 2), 8), ("1x7", (1, 7), (1, 1), (0, 3), 12),
          ("7x1", (7, 1), (1, 1), (3, 0), 12), ("1x3", (1, 3), (1, 1), (0, 1), 8), ("3x1", (3, 1), (1, 1), (1, 0), 8),
          ("11x11/4 stem", (11, 11), (4, 4), (2, 2), 3), ("3x3/2 stem", (3, 3), (2, 2), (0, 0), 3)]


@pytest.mark.parametrize("what,kernel,stride,padding,ci", SHAPES, ids=[s[0] for s in SHAPES])
def test_fp32_packing_against_conv2d(what, kernel, stride, padding, ci):
    from ladi_vton_b200.metrics import fold_bn, pack_im2col_weight, pad4
    g = torch.Generator().manual_seed(31)
    co = 20
    w = torch.randn(co, ci, *kernel, generator=g, dtype=torch.float64)
    gamma, beta = torch.rand(co, generator=g, dtype=torch.float64) + 0.5, torch.randn(co, generator=g, dtype=torch.float64)
    mean, var = torch.randn(co, generator=g, dtype=torch.float64), torch.rand(co, generator=g, dtype=torch.float64) + 0.5
    x = torch.randn(2, ci, 23, 19, generator=g, dtype=torch.float64)
    ref = F.batch_norm(F.conv2d(x, w, None, stride, padding), mean, var, gamma, beta, False, 0.0, 1e-3)
    wf, bf = fold_bn(w, gamma, beta, mean, var, 1e-3)
    packed = pack_im2col_weight(wf, torch.float32)
    k = kernel[0] * kernel[1] * ci
    assert packed.dtype == torch.float32 and packed.is_contiguous() and packed.shape == (co, pad4(k)) and pad4(k) % 4 == 0
    assert pad4(k) - k < 4 and bool((packed[:, k:] == 0).all())
    # the fold happened in float64: the packed values are the float64 folded weights rounded once to fp32
    assert torch.equal(packed[:, :k], wf.permute(0, 2, 3, 1).reshape(co, k).float())
    rows, (n, oh, ow) = _im2col_rows(x, kernel, stride, padding, packed.shape[1])
    got = (rows @ packed.double().T + bf).view(n, oh, ow, co).permute(0, 3, 1, 2)
    mag = F.conv2d(x.abs(), w.abs() * (gamma / torch.sqrt(var + 1e-3)).view(-1, 1, 1, 1), None, stride, padding)
    assert float(((got - ref).abs() - 2.0 ** -24 * mag).max()) <= 1e-12  # one fp32 rounding of each weight


def test_precision_rejects_unknown():
    from ladi_vton_b200.metrics import FIDInceptionV3, LPIPSAlex
    assert FIDInceptionV3().precision == "bf16" and LPIPSAlex().precision == "bf16"
    assert FIDInceptionV3("tf32").dtype == torch.float32 and LPIPSAlex(precision="tf32").dtype == torch.float32
    for cls in (FIDInceptionV3, LPIPSAlex):
        with pytest.raises(ValueError, match="precision"):
            cls("fp16")


# ---- CLI --------------------------------------------------------------------------------------------------------------------------------
def test_cli_parser_adds_precision_to_the_engine_group():
    """main()'s parser is build_parser() (the reference's flags plus the offline options) with --precision in its engine group, nothing else."""
    from ladi_vton_b200.val_metrics import build_cli_parser, build_parser

    def flags(parser):
        groups = {g.title: {a.option_strings[0] for a in g._group_actions if a.option_strings} for g in parser._action_groups}
        return {a.option_strings[0] for a in parser._actions if a.option_strings}, groups.get("engine", set())
    base_all, base_eng = flags(build_parser())
    cli_all, cli_eng = flags(build_cli_parser())
    assert cli_all - base_all == {"--precision"} and base_all <= cli_all
    assert cli_eng == base_eng | {"--precision"}
    act = next(a for a in build_cli_parser()._actions if "--precision" in a.option_strings)
    assert act.default == "bf16" and list(act.choices) == ["bf16", "tf32"]


def test_precision_flag():
    from ladi_vton_b200.val_metrics import build_cli_parser
    base = ["--gen_folder", "g", "--test_order", "paired", "--dataset", "vitonhd"]
    p = build_cli_parser()
    assert p.parse_args(base).precision == "bf16"
    assert p.parse_args(base + ["--precision", "tf32"]).precision == "tf32"
    assert p.parse_args(base + ["--precision", "bf16"]).precision == "bf16"
    with pytest.raises(SystemExit):
        p.parse_args(base + ["--precision", "fp32"])


def test_weights_tag_names_the_precision(tmp_path):
    from ladi_vton_b200.metrics import INCEPTION_FILE
    from ladi_vton_b200.val_metrics import weights_tag
    assert weights_tag(None, 0, True) == weights_tag(None, 0, True, "bf16") == "random0"  # the bf16 cache files keep their names
    assert weights_tag(None, 0, True, "tf32") not in (weights_tag(None, 0, True), weights_tag(None, 1, True, "tf32"))
    (tmp_path / INCEPTION_FILE).write_bytes(b"\0" * 10)
    bf, tf = weights_tag(str(tmp_path), 0, False), weights_tag(str(tmp_path), 0, False, "tf32")
    assert bf == weights_tag(str(tmp_path), 0, False, "bf16") and tf != bf and bf in tf


# ---- census of the recorded tf32 calls ----------------------------------------------------------------------------------------------
GEMM_ARGS = "a m k a_pitch w n w_pitch bias relu out out_pitch c_off stream".split()


def tf32_calls(B, H=512, W=384):
    """The ABI calls of FIDInceptionV3 (FID features and is_features) and LPIPSAlex at batch B, tf32, recorded on the CPU."""
    from ladi_vton_b200.metrics import FIDInceptionV3, LPIPSAlex, random_state_dict
    inc, lp = FIDInceptionV3("tf32"), LPIPSAlex("tf32")
    inc = cpu_pack(inc, random_state_dict(inc.param_shapes(), 0))
    lp = cpu_pack(lp, random_state_dict(lp.param_shapes(), 1))

    def run():
        inc(torch.zeros((B, 3, 299, 299)))
        inc.is_features(torch.zeros((B, 3, H, W)))
        lp(torch.zeros((B, 3, H, W)), torch.zeros((B, 3, H, W)))
    return recorded(run)


@pytest.mark.parametrize("B", [1, 8, 32])
def test_tf32_census_placements(B):
    calls = tf32_calls(B)
    names = {n for n, _ in calls}
    assert names == {"ladi_gemm_tf32", "ladi_im2col_f32", "ladi_pool2d_f32", "ladi_lpips_layer_f32", "ladi_resize_tf1_u8"}, names
    gemms = [dict(zip(GEMM_ARGS, args)) for n, args in calls if n == "ladi_gemm_tf32"]
    # 94 Inception convolutions twice (FID features, IS features), 5 AlexNet convolutions
    assert len(gemms) == 2 * 94 + 5
    widths = set()
    for g in gemms:
        # CPU tensors from the 64-byte aligned allocator: an address that is a multiple of 16 here is one on the device
        assert g["a"].value % 16 == 0 and g["w"].value % 16 == 0 and g["out"].value % 16 == 0, g
        assert g["a_pitch"] % 4 == 0 and g["w_pitch"] % 4 == 0 and g["a_pitch"] >= g["k"] and g["w_pitch"] >= g["k"], g
        assert g["n"] % 4 == 0 and g["c_off"] % 4 == 0 and g["out_pitch"] % 4 == 0 and g["c_off"] + g["n"] <= g["out_pitch"], g
        assert g["relu"] == 1 and g["bias"].value and (g["m"] + 127) // 128 <= 65535, g
        widths.add(g["n"])
    assert widths == {32, 48, 64, 80, 96, 128, 160, 192, 256, 320, 384, 448}
    assert any(g["c_off"] and g["out_pitch"] == 2048 for g in gemms), "branch outputs into the Mixed_7 concatenations"
    assert any(g["k"] % 32 for g in gemms), "reductions that end inside a 32-column block"
