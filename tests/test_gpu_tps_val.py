"""GPU tests of the warping trainer's validation on the engine (vgg.py, eval_tps.py <- src/utils/vgg_loss.py, src/train_tps.py:29-92):
  * `ladi_l1_mean_f32` against float64 at its edges (one element, counts that are not a multiple of the block or of 4, a pitch past the
    width with NaN-poisoned padding, one 16 x 3 x 512 x 384 image pair), within the accumulation bound C_ACC sqrt(n) 2^-24 sum|a - b| plus
    one fp32 rounding, and bit-identical when run twice;
  * the fp32 forms of resize_aa and warp_grid_sample within the float64 bounds of tests/kernel_check.py (u_out = 2^-24), and their bf16
    forms equal to the round-to-nearest bf16 of the fp32 forms on the same inputs, bit for bit;
  * the VGG-19 taps and the loss against the fp32 oracle with TF32 off: the engine's relative error at most 1.5 times that of cuDNN's own
    TF32 run of the oracle (tap 1: 2^-10 instead, as cuDNN computes the 3-channel first convolution in plain fp32; the loss: or 1e-4);
  * compute_metric end to end at 512 x 384, batch 16, full-width random weights, TPS-only and with refinement, dense and not, against the
    fp32 oracle body;
  * `main()` on synthetic samples: the JSON, and the same bits from two runs;
  * the census: every distinct kernel call of one validation batch (TPS-only and with refinement, dense and not, batch 1 and 16, 512x384),
    recorded on the CPU and replayed against float64 with per-element bounds on the shared harness of tests/kernel_check.py.  The bf16
    warping calls go through the glue census's classification and replays (kernel_check.glue_collect / REPLAY); the fp32 calls through
    the replays below.  Their bounds (u = 2^-24): ladi_gemm_tf32 U_F32 |r| + (2^-10 + C_ACC sqrt(K) u) (|A| |W|^T + |bias|) (operands
    rounded to nearest TF32, fp32 sum), as tests/test_gpu_metrics_tf32.py derives it; im2col NHWC and max pool exact; the pixel im2col
    bit-equal to torch's fp32 (x - shift) / scale; resize_aa_f32 / warp_grid_sample_f32 kernel_check's resample / warp bounds with
    u_out = u; l1_mean_f32 w C_ACC sqrt(n) u S / n + u (w S / n) + u |r| with S = sum|a - b|, r = acc + w S / n.  Every replay also checks
    that the call wrote only its own elements (NaN-poisoned pitch gaps and tails stay NaN, poisoned inputs are never read) and that two runs
    give the same bits.
"""
import importlib.util
import json
import math
import os

import pytest
import torch

from kernel_check import (C_ACC, EPS24, REPLAY, U_F32, Replay, cpu_pack, determinism, flat_buf, glue_collect, key_of, layout, ptr, recorded,
                          rel_l2, resample_expect, tail_nan, twice, warp_expect, worst_at)

pytestmark = pytest.mark.gpu


def _l1_call(a, b, rows, cols, a_pitch, b_pitch, weight, dev):
    from ladi_vton_b200 import lib, ops
    acc = torch.full((1,), 0.0, dtype=torch.float32, device=dev)
    ws = torch.empty(ops.L1_MEAN_WS, dtype=torch.float32, device=dev)
    lib.call("ladi_l1_mean_f32", ops._ptr(a), a_pitch, ops._ptr(b), b_pitch, rows, cols, float(weight), ops._ptr(ws), ops._ptr(acc),
             ops._stream())
    torch.cuda.synchronize()
    return acc


@pytest.mark.parametrize("rows,cols,a_pitch,b_pitch,weight", [
    (1, 1, 1, 1, 1.0), (1, 3, 4, 5, 0.25), (7, 13, 16, 13, 1.0 / 32), (1000, 1001, 1001, 1001, 1.0), (257, 64, 64, 64, 1.0 / 16),
    (4099, 100, 104, 112, 0.125), (16 * 3 * 512, 384, 384, 384, 1.0)])
def test_l1_mean_against_float64(cuda, rows, cols, a_pitch, b_pitch, weight):
    g = torch.Generator().manual_seed(rows * 7 + cols)
    a = torch.full((rows, a_pitch), float("nan"))
    b = torch.full((rows, b_pitch), float("nan"))
    a[:, :cols] = torch.randn((rows, cols), generator=g)
    b[:, :cols] = torch.randn((rows, cols), generator=g) * 0.5
    ad, bd = a.to(cuda), b.to(cuda)
    y = _l1_call(ad, bd, rows, cols, a_pitch, b_pitch, weight, cuda)
    y2 = _l1_call(ad, bd, rows, cols, a_pitch, b_pitch, weight, cuda)
    assert torch.equal(y, y2)
    n = rows * cols
    s = (a[:, :cols].double() - b[:, :cols].double()).abs().sum().item()
    r = weight * s / n
    bound = weight * C_ACC * math.sqrt(n) * EPS24 * s / n + EPS24 * abs(r)
    err = abs(y.item() - r)
    print(f"\nl1_mean {rows}x{cols} (pitches {a_pitch}, {b_pitch}): |err| {err:.3e}, bound {bound:.3e}")
    assert math.isfinite(y.item()) and err <= bound


def test_l1_mean_accumulates_and_wrapper(cuda):
    from ladi_vton_b200 import ops
    g = torch.Generator().manual_seed(1)
    a, b = torch.randn((3, 5, 6), generator=g), torch.randn((3, 5, 6), generator=g)
    acc = torch.full((1,), 0.5, device=cuda)
    ops.l1_mean_(a.to(cuda), b.to(cuda), acc, 0.25)
    r = 0.5 + 0.25 * float((a.double() - b.double()).abs().mean())
    assert abs(acc.item() - r) <= 4 * EPS24 * r


@pytest.mark.parametrize("h,w,oh,ow", [(512, 384, 341, 256), (256, 192, 341, 256), (512, 384, 256, 192), (37, 29, 11, 7)])
def test_resize_aa_f32_and_bf16_form(cuda, h, w, oh, ow):
    from ladi_vton_b200 import ops
    x = torch.rand((2, 3, h, w), generator=torch.Generator().manual_seed(h), dtype=torch.float32) * 2 - 1
    xd = x.to(cuda)
    y = ops.resize_aa_f32(xd, oh, ow)
    r, bound = resample_expect(xd.double(), oh, ow, EPS24)
    q = ((y.double() - r).abs() / bound).max().item()
    print(f"\nresize_aa_f32 {h}x{w} -> {oh}x{ow}: worst err/bound {q:.3f}")
    assert q <= 1
    assert torch.equal(ops.resize_aa_f32(xd, oh, ow), y)
    yb = ops.resize_aa(xd, oh, ow)  # NHWC bf16, pitch 8
    assert torch.equal(yb[..., :3], y.permute(0, 2, 3, 1).to(torch.bfloat16))


@pytest.mark.parametrize("gh,gw,H,W", [(256, 192, 512, 384), (256, 192, 256, 192), (64, 48, 100, 70)])
def test_warp_grid_sample_f32_and_bf16_form(cuda, gh, gw, H, W):
    from ladi_vton_b200 import ops, synthetic as S
    g = torch.Generator().manual_seed(gh + H)
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, gh), torch.linspace(-1, 1, gw), indexing="ij")
    grid = torch.stack([xs, ys], -1)[None].repeat(2, 1, 1, 1) * 1.05 + torch.randn((2, gh, gw, 2), generator=g) * 0.02
    cloth = S.warp_inputs(2, H, W, seed=gh)["cloth"]
    gd, cd = grid.contiguous().to(cuda), cloth.contiguous().to(cuda)
    y = ops.warp_grid_sample_f32(gd, cd)
    r, bound = warp_expect(gd.double(), cd.double(), EPS24)
    q = ((y.double() - r).abs() / bound).max().item()
    print(f"\nwarp_grid_sample_f32 {gh}x{gw} -> {H}x{W}: worst err/bound {q:.3f}")
    assert q <= 1
    out = torch.zeros((2, H, W, 8), dtype=torch.bfloat16, device=cuda)
    ops.warp_grid_sample(gd, cd, out, c_off=2)
    assert torch.equal(out[..., 2:5], y.permute(0, 2, 3, 1).to(torch.bfloat16))
    assert not out[..., :2].any() and not out[..., 5:].any()


def _tf32(flag, fn):
    """fn() with cuDNN's TF32 convolutions on or off (matmuls stay fp32, PyTorch's default), as test_gpu_metrics_tf32.py runs its oracle."""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = flag
    try:
        return fn()
    finally:
        torch.backends.cudnn.allow_tf32 = old


def _generator():
    """tests/golden/make_tps_val_golden.py, for its seeded VGG weights (non-zero biases)."""
    spec = importlib.util.spec_from_file_location("make_tps_val_golden", os.path.join(os.path.dirname(__file__), "golden", "make_tps_val_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _vgg_pair(cuda, seed=181):
    from ladi_oracle.vgg import VGG19 as OV, VGGLoss as OL
    from ladi_vton_b200.vgg import VGGLoss
    sd = _generator().vgg_state_dict(seed)
    assert all(bool((v != 0).all()) for k, v in sd.items() if k.endswith(".bias"))
    return VGGLoss().load_state_dict(sd).to(cuda), OL(OV().load_torchvision(sd)).to(cuda).eval()


@pytest.mark.parametrize("B,H,W", [(2, 512, 384), (16, 512, 384), (3, 256, 192)])
def test_vgg_taps_and_loss_against_oracle(cuda, B, H, W):
    from ladi_vton_b200 import ops
    from ladi_vton_b200.vgg import resized_size
    eng, orc = _vgg_pair(cuda)
    g = torch.Generator().manual_seed(B)
    x = (torch.rand((B, 3, H, W), generator=g) * 2 - 1).to(cuda)
    y = (x.cpu() * 0.7 + (torch.rand((B, 3, H, W), generator=g) * 2 - 1) * 0.3).to(cuda)
    with torch.no_grad():
        oh, ow = resized_size(H, W)
        xy = torch.cat([ops.resize_aa_f32(x, oh, ow), ops.resize_aa_f32(y, oh, ow)])
        taps = eng.vgg.taps(xy)
        prep = torch.cat([orc.prepare(x), orc.prepare(y)])
        ref = _tf32(False, lambda: orc.vgg(prep))
        cud = _tf32(True, lambda: orc.vgg(prep))
        for i, (t, r, c) in enumerate(zip(taps, ref, cud)):
            e, ec = rel_l2(t.permute(0, 3, 1, 2), r), rel_l2(c, r)
            print(f"\n[vgg {B}x{H}x{W}] tap {i + 1}: engine rel-L2 {e:.3e}, cuDNN TF32 {ec:.3e}")
            if i == 0:  # cuDNN computes the 3-channel conv1_1 in plain fp32 (its TF32 run is exact): TF32's product bound 2^-10
                assert e <= 2.0 ** -10
            else:
                assert 0 < ec and e <= 1.5 * ec
        loss = eng(x, y).item()
        lr = _tf32(False, lambda: orc(x, y)).item()
        lc = _tf32(True, lambda: orc(x, y)).item()
    el, ecl = abs(loss - lr) / abs(lr), abs(lc - lr) / abs(lr)
    print(f"[vgg {B}x{H}x{W}] loss {loss:.6f} vs fp32 {lr:.6f}: rel {el:.2e} (cuDNN TF32 {ecl:.2e})")
    assert el <= max(1.5 * ecl, 1e-4)
    assert eng(x, y).item() == loss
    if B == 16:
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        eng(x, y)
        torch.cuda.synchronize()
        print(f"[vgg {B}x{H}x{W}] peak memory above the inputs: {(torch.cuda.max_memory_allocated() - base) / 2 ** 20:.0f} MiB")


def _warp_models(cuda, dense, seed=61):
    from ladi_oracle.warp import ConvNet_TPS as OT, UNetVanilla as OU
    from ladi_vton_b200 import synthetic as S
    from ladi_vton_b200.warp import ConvNet_TPS, UNetVanilla, control_points
    tps, ref = ConvNet_TPS(256, 192, 5 if dense else 21, 3), UNetVanilla(8 if dense else 24, 3, bilinear=True)
    tsd = S.warp_state_dict(tps.param_shapes(), seed, ctrl_bias=torch.atanh(control_points()).view(-1))
    rsd = S.warp_state_dict(ref.param_shapes(), seed + 10)
    ot, ou = OT(256, 192, 5 if dense else 21, 3).eval(), OU(8 if dense else 24, 3).eval()
    ot.load_state_dict(tsd, strict=False)
    ou.load_state_dict(rsd)
    return tps.load_state_dict(tsd).to(cuda), ref.load_state_dict(rsd).to(cuda), ot.to(cuda), ou.to(cuda)


def _batches(n_batches, B, H, W, dense, seed):
    from ladi_vton_b200.eval_tps import OUTPUTLIST
    from ladi_vton_b200.inference import SyntheticTryOnDataset
    ds = SyntheticTryOnDataset(n_batches * B, (H, W), seed=seed, outputlist=OUTPUTLIST + (["dense_uv"] if dense else []))
    return [torch.utils.data.default_collate([ds[k * B + i] for i in range(B)]) for k in range(n_batches)]


@pytest.mark.parametrize("dense", [False, True])
@pytest.mark.parametrize("stage", ["tps", "refinement"])
def test_compute_metric_end_to_end(cuda, dense, stage):
    """512 x 384, batch 16, two batches: the engine's (loss, vgg_loss) against the fp32 oracle body on the GPU, TF32 off."""
    from ladi_oracle.tps_val_body import compute_metric as oracle_metric
    from ladi_vton_b200.eval_tps import compute_metric
    from ladi_vton_b200.vgg import L1Loss
    tps, ref, ot, ou = _warp_models(cuda, dense)
    vgg, ovgg = _vgg_pair(cuda)
    batches = _batches(2, 16, 512, 384, dense, 5)
    loss, vloss, visual = compute_metric(batches, tps, L1Loss(), vgg, refinement=ref if stage == "refinement" else None)
    dev_b = [{k: (v.to(cuda) if torch.is_tensor(v) else v) for k, v in b.items()} for b in batches]
    rl, rv, _ = _tf32(False, lambda: oracle_metric(dev_b, ot, ovgg, ou if stage == "refinement" else None))
    el, ev = abs(loss - rl) / abs(rl), abs(vloss - rv) / abs(rv)
    print(f"\n[tps val {stage} dense={dense}] L1 {loss:.6f} vs {rl:.6f} (rel {el:.2e}); VGG {vloss:.6f} vs {rv:.6f} (rel {ev:.2e})")
    assert len(visual[0]) == 4 and float(visual[0][3].abs().max()) <= 1
    assert el <= 1e-2 and ev <= 2e-2
    l2, v2, _ = compute_metric(batches, tps, L1Loss(), vgg, refinement=ref if stage == "refinement" else None)
    assert (l2, v2) == (loss, vloss)
    _, z, _ = compute_metric(batches[:1], tps, L1Loss(), None, refinement=None)
    assert z == 0


def test_cli_main_synthetic(cuda, tmp_path):
    from ladi_vton_b200.eval_tps import main
    argv = ["--dataset", "vitonhd", "--exp_name", "e", "--synthetic_samples", "8", "-b", "4", "--random_init"]
    r1 = main(argv + ["--output_json", str(tmp_path / "a.json")])
    r2 = main(argv + ["--output_json", str(tmp_path / "b.json")])
    out = json.load(open(tmp_path / "a.json"))
    assert list(out) == ["epoch", "stage", "eval/eval_loss_paired", "eval/eval_vgg_loss_paired", "eval/eval_loss_unpaired",
                         "eval/eval_vgg_loss_unpaired"]
    assert out["epoch"] == 0 and out["stage"] == "tps" and all(math.isfinite(out[k]) and out[k] > 0 for k in list(out)[2:])
    assert r1 == r2 == out
    r3 = main(argv + ["--stage", "refinement", "--vgg_weight", "0", "--dense"])
    assert r3["stage"] == "refinement" and r3["eval/eval_vgg_loss_paired"] == 0 and r3["eval/eval_loss_paired"] > 0


# ================================================================================================================ census replay
E_TF32 = 2.0 ** -10  # both operands rounded to nearest TF32 inside ladi_gemm_tf32
FP32_ARGS = {"ladi_gemm_tf32": ("gemm_tf32", "a m k a_pitch wt n w_pitch bias relu out out_pitch c_off stream"),
             "ladi_im2col_f32": ("im2col_f32", "x pixels n c h w pitch kh kw sh sw ph pw shift scale out kpad stream"),
             "ladi_pool2d_f32": ("pool2d_f32", "x n h w c xp k s p mode out op c_off stream"),
             "ladi_resize_aa_f32": ("resize_aa_f32", "x n c h w oh ow out stream"),
             "ladi_warp_grid_sample_f32": ("warp_grid_sample_f32", "grid gh gw cloth n c H W out stream"),
             "ladi_l1_mean_f32": ("l1_mean_f32", "a ap b bp rows cols weight ws acc stream")}
POINTERS = {"a", "wt", "bias", "out", "stream", "x", "shift", "scale", "grid", "cloth", "b", "ws", "acc"}
CENSUS_BATCHES = (1, 16)


def _lib():
    from ladi_vton_b200 import lib
    return lib


def _f32(R, rows, pitch, values):
    return R.poisoned(rows, pitch, values, dtype=torch.float32)


def replay_gemm_tf32(R, f, chunk=1 << 18):
    m, k, ap, n, wp, op, c_off, relu = (f[q] for q in ("m", "k", "a_pitch", "n", "w_pitch", "out_pitch", "c_off", "relu"))
    a = _f32(R, m, ap, R.randn(m, k) * 2.0)
    w = _f32(R, n, wp, R.randn(n, k) / math.sqrt(k))
    b = R.randn(n) * 0.5

    def fresh():
        flat, o = flat_buf(R, m * op, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda bf: _lib().call("ladi_gemm_tf32", ptr(a), m, k, ap, ptr(w), n, wp, ptr(b), relu, ptr(bf["out"]), op, c_off, R.stream),
                 fresh)
    out = runs[0]["out"].view(m, op)
    errs = layout(out, c_off, c_off + n, "out") + tail_nan(runs[0]["flat"], m * op, "out") + determinism(runs, ["flat"])
    W, B = w[:, :k].double(), b.double()
    worst = (0.0, "")
    for r0 in range(0, m, chunk):
        A = a[r0:r0 + chunk, :k].double()
        pre = A @ W.T + B
        r = pre.clamp_min(0) if relu else pre
        bound = U_F32 * r.abs() + (E_TF32 + C_ACC * math.sqrt(k) * EPS24) * (A.abs() @ W.abs().T + B.abs())
        q = torch.nan_to_num((out[r0:r0 + chunk, c_off:c_off + n].double() - r).abs() / bound.clamp_min(1e-300), nan=float("inf"))
        e, res = worst_at(q, ("row", "column"), f" (rows from {r0}; m {m} n {n} k {k})")
        errs += e
        worst = max(worst, res)
    return errs, worst


def _im2col_ref(x, kh, kw, sh, sw, ph, pw, k_pad):
    """x NHWC [n, h, w, c] -> rows [n*oh*ow, k_pad], column (ky*kw + kx)*c + ch, zeros in the padding and in columns >= kh*kw*c."""
    n, h, w, c = x.shape
    oh, ow = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
    xp = torch.nn.functional.pad(x, (0, 0, pw, pw, ph, ph))
    taps = [xp[:, ky:ky + sh * (oh - 1) + 1:sh, kx:kx + sw * (ow - 1) + 1:sw, :] for ky in range(kh) for kx in range(kw)]
    return torch.nn.functional.pad(torch.stack(taps, dim=3).reshape(n * oh * ow, kh * kw * c), (0, k_pad - kh * kw * c))


def replay_im2col_f32(R, f):
    from ladi_vton_b200.vgg import MEAN, STD
    n, c, h, w, pitch, kh, kw, sh, sw, ph, pw, kp = (f[q] for q in ("n", "c", "h", "w", "pitch", "kh", "kw", "sh", "sw", "ph", "pw", "kpad"))
    oh, ow = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
    rows = n * oh * ow
    geo = (kh, kw, sh, sw, ph, pw, kp)
    if f["pixels"]:  # VGGLoss's normalisation of [-1, 1] images
        x = R.rand(n, c, h, w) * 2 - 1
        shift = torch.tensor([2 * m - 1 for m in MEAN], device=R.dev)
        scale = torch.tensor([2 * s for s in STD], device=R.dev)
    else:
        x, shift, scale = _f32(R, n * h * w, pitch, R.randn(n * h * w, c).clamp_min(0.0)), None, None

    def fresh():
        flat, o = flat_buf(R, rows * kp, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: _lib().call("ladi_im2col_f32", ptr(x), int(f["pixels"]), n, c, h, w, pitch, kh, kw, sh, sw, ph, pw, ptr(shift),
                                       ptr(scale), ptr(b["out"]), kp, R.stream), fresh)
    out = runs[0]["out"].view(rows, kp)
    errs = layout(out, 0, kp, "rows") + tail_nan(runs[0]["flat"], rows * kp, "rows") + determinism(runs, ["flat"])
    if f["pixels"]:
        q = (x - shift.view(-1, 1, 1)) / scale.view(-1, 1, 1)  # torch fp32, IEEE division
        ok = torch.equal(out, _im2col_ref(q.permute(0, 2, 3, 1), *geo))
    else:
        ok = torch.equal(out, _im2col_ref(x.view(n, h, w, pitch)[..., :c], *geo))
    return errs + ([] if ok else ["im2col differs from the exact rows"]), (0.0, "exact")


def replay_pool2d_f32(R, f):
    n, h, w, c, xp, k, s, p, mode, op, c_off = (f[q] for q in ("n", "h", "w", "c", "xp", "k", "s", "p", "mode", "op", "c_off"))
    assert mode == 0, "VGG-19 pools are max pools"
    x = _f32(R, n * h * w, xp, R.randn(n * h * w, c) * 2.0)
    X = x[:, :c].reshape(n, h, w, c).permute(0, 3, 1, 2)
    oh, ow = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    rows = n * oh * ow

    def fresh():
        flat, o = flat_buf(R, rows * op, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: _lib().call("ladi_pool2d_f32", ptr(x), n, h, w, c, xp, k, s, p, mode, ptr(b["out"]), op, c_off, R.stream), fresh)
    out = runs[0]["out"].view(rows, op)
    errs = layout(out, c_off, c_off + c, "output") + tail_nan(runs[0]["flat"], rows * op, "output") + determinism(runs, ["flat"])
    r = torch.nn.functional.max_pool2d(X, k, s, p).permute(0, 2, 3, 1).reshape(rows, c)
    return errs + ([] if torch.equal(out[:, c_off:c_off + c], r) else ["max pool is not exact"]), (0.0, "exact")


def replay_resize_aa_f32(R, f):
    n, c, h, w, oh, ow = (f[q] for q in ("n", "c", "h", "w", "oh", "ow"))
    x = R.rand(n, c, h, w) * 2 - 1

    def fresh():
        flat, o = flat_buf(R, n * c * oh * ow, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: _lib().call("ladi_resize_aa_f32", ptr(x), n, c, h, w, oh, ow, ptr(b["out"]), R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], n * c * oh * ow, "out") + determinism(runs, ["flat"])
    r, bound = resample_expect(x.double(), oh, ow, EPS24)
    q = torch.nan_to_num((runs[0]["out"].view(n, c, oh, ow).double() - r).abs() / bound.clamp_min(1e-300), nan=float("inf"))
    e, res = worst_at(q, ("image", "channel", "y", "x"))
    return errs + e, res


def replay_warp_grid_sample_f32(R, f):
    gh, gw, n, c, H, W = (f[q] for q in ("gh", "gw", "n", "c", "H", "W"))
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, gh, device=R.dev), torch.linspace(-1, 1, gw, device=R.dev), indexing="ij")
    grid = (torch.stack([xs, ys], -1)[None] * 1.05 + R.randn(n, gh, gw, 2) * 0.02).contiguous()  # past the border too
    cloth = R.rand(n, c, H, W) * 2 - 1

    def fresh():
        flat, o = flat_buf(R, n * c * H * W, torch.float32)
        return dict(flat=flat, out=o)
    runs = twice(lambda b: _lib().call("ladi_warp_grid_sample_f32", ptr(grid), gh, gw, ptr(cloth), n, c, H, W, ptr(b["out"]), R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], n * c * H * W, "out") + determinism(runs, ["flat"])
    r, bound = warp_expect(grid.double(), cloth.double(), EPS24)
    q = torch.nan_to_num((runs[0]["out"].view(n, c, H, W).double() - r).abs() / bound.clamp_min(1e-300), nan=float("inf"))
    e, res = worst_at(q, ("image", "channel", "y", "x"))
    return errs + e, res


def replay_l1_mean_f32(R, f):
    from ladi_vton_b200 import ops
    ap, bp, rows, cols, weight = (f[q] for q in ("ap", "bp", "rows", "cols", "weight"))
    a = _f32(R, rows, ap, R.randn(rows, cols).clamp_min(0.0))
    b = _f32(R, rows, bp, R.randn(rows, cols).clamp_min(0.0))
    acc0 = float(R.rand(1)) + 0.25

    def fresh():
        wflat, ws = flat_buf(R, ops.L1_MEAN_WS, torch.float32)
        flat, acc = flat_buf(R, 1, torch.float32)
        acc.fill_(acc0)
        return dict(flat=flat, acc=acc, wflat=wflat, ws=ws)
    runs = twice(lambda bf: _lib().call("ladi_l1_mean_f32", ptr(a), ap, ptr(b), bp, rows, cols, float(weight), ptr(bf["ws"]), ptr(bf["acc"]),
                                        R.stream), fresh)
    errs = tail_nan(runs[0]["flat"], 1, "acc") + tail_nan(runs[0]["wflat"], ops.L1_MEAN_WS, "ws") + determinism(runs, ["flat"])
    nel = rows * cols
    S = (a[:, :cols].double() - b[:, :cols].double()).abs().sum().item()
    term = weight * S / nel
    r = acc0 + term
    bound = weight * C_ACC * math.sqrt(nel) * EPS24 * S / nel + EPS24 * term + EPS24 * abs(r)
    y = runs[0]["acc"].item()
    q = abs(y - r) / bound if math.isfinite(y) else float("inf")
    return errs + ([f"err/bound {q:.3g}"] if q > 1 else []), (q, f"rows {rows} cols {cols}")


FP32_REPLAY = {"gemm_tf32": replay_gemm_tf32, "im2col_f32": replay_im2col_f32, "pool2d_f32": replay_pool2d_f32,
               "resize_aa_f32": replay_resize_aa_f32, "warp_grid_sample_f32": replay_warp_grid_sample_f32, "l1_mean_f32": replay_l1_mean_f32}


def _validation_calls(B, dense, stage):
    """The ABI calls of compute_metric on one 512x384 batch of B pairs, recorded on the CPU (weights packed on the CPU, nothing launched)."""
    from ladi_vton_b200 import synthetic as S
    from ladi_vton_b200.eval_tps import compute_metric
    from ladi_vton_b200.metrics import random_state_dict
    from ladi_vton_b200.vgg import VGG19, L1Loss, VGGLoss
    from ladi_vton_b200.warp import ConvNet_TPS, UNetVanilla
    tps, ref = ConvNet_TPS(256, 192, 5 if dense else 21, 3), UNetVanilla(8 if dense else 24, 3, bilinear=True)
    cpu_pack(tps, S.warp_state_dict(tps.param_shapes(), 13))
    cpu_pack(ref, S.warp_state_dict(ref.param_shapes(), 14))
    vgg = VGGLoss(cpu_pack(VGG19(), random_state_dict(VGG19().param_shapes(), 15)))
    z = lambda c: torch.zeros((B, c, 512, 384))  # noqa: E731
    batch = dict(image=z(3), cloth=z(3), im_cloth=z(3), im_mask=z(3), pose_map=z(18))
    if dense:
        batch["dense_uv"] = z(2)
    return recorded(lambda: compute_metric([batch], tps, L1Loss(), vgg, refinement=ref if stage == "refinement" else None))


def tps_val_census():
    """-> {key: (kind, fields, first workload, replay)} over CENSUS_BATCHES x (tps, refinement) x (dense or not)."""
    desc, rest = {}, []
    for B in CENSUS_BATCHES:
        for stage in ("tps", "refinement"):
            for dense in (False, True):
                label = f"B={B} {stage}{' dense' if dense else ''}"
                calls = _validation_calls(B, dense, stage)
                other = []
                for name, args in calls:
                    if name in FP32_ARGS:
                        kind, spec = FP32_ARGS[name]
                        f = {k: (float(v) if k == "weight" else int(v)) for k, v in zip(spec.split(), args) if k not in POINTERS}
                        desc.setdefault(key_of(kind, f), (kind, f, label, FP32_REPLAY[kind]))
                    else:
                        other.append((name, args))
                rest.append((label, other))
    gdesc, _, unknown = glue_collect([(label, (lambda o=o: o)) for label, o in rest])
    assert not unknown, unknown
    for key, d in gdesc.items():
        desc.setdefault(key, (d["kind"], d["f"], d["first"], REPLAY[d["kind"]]))
    return desc


def test_tps_val_census_replay_against_float64(cuda):
    desc = tps_val_census()
    kinds = {}
    for kind, f, _, _ in desc.values():
        kinds.setdefault(kind, []).append(f)
    print(f"\n[tps val census] {len(desc)} distinct calls over batches {CENSUS_BATCHES}: "
          + ", ".join(f"{k} {len(v)}" for k, v in sorted(kinds.items())))
    # what the census must hold: the 13 VGG convolutions' (K, N), the four pools on 341 / 170 / 85 / 42 rows, tap- and image-shaped L1
    from ladi_vton_b200.vgg import CONVS
    assert {(f["k"], f["n"]) for f in kinds["gemm_tf32"]} == {((9 * ci + 3) // 4 * 4, co) for ci, co in CONVS.values()}
    assert {f["h"] for f in kinds["pool2d_f32"]} == {341, 170, 85, 42}
    assert {f["cols"] for f in kinds["l1_mean_f32"]} >= {384, 64, 128, 256, 512}
    assert {"resize_aa_f32", "warp_grid_sample_f32", "conv", "resize_aa", "warp_grid_sample", "tps_grid"} <= set(kinds)
    R = Replay(cuda, 24680)
    bad, worst = [], {}
    for key, (kind, f, first, replay) in desc.items():
        errs, res = replay(R, f)
        bad += [f"{key} (first in {first}): {e}" for e in errs[:2]]
        if res is not None:
            worst[kind] = max(worst.get(kind, (0.0, "")), (res[0], f"{key}: {res[1]}"))
        torch.cuda.empty_cache()
    for k, (w, where) in sorted(worst.items()):
        print(f"  {k}: worst err/bound {w:.3f} at {where}")
    assert not bad, "\n".join(bad[:10])
