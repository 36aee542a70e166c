"""GPU tests of the EMASC trainer's validation on the engine (`eval.extract_save_vae_images`, `python -m ladi_vton_b200.eval_emasc`):
  * `ladi_image_save_u8` bit for bit against torchvision save_image's expression on the CPU,
    `x.add(1).div(2).mul(255).add_(0.5).clamp_(0, 255).to(uint8)`, over every fp32 value within 64 ulps of each of the 256 rounding
    boundaries, 10^6 random values in [-1.2, 1.2], +-1, +-inf and values out of range, with the input's pad channel NaN-poisoned; NaN
    gives 0, nothing past the output is written, and a second run is bit-identical;
  * the reconstruction body (`vae_recon_batch`) at the small VAE config against the fp32 oracle body on the GPU with the same seeded CUDA
    RNG, for the three EMASC forms and without EMASC, at the gates of test_gpu_models.py::test_train_emasc_forward_small;
  * the full-size VAE and nonlinear 3x3 EMASC at batch 16, 512x384, per image against the fp32 oracle on the GPU (TF32 off);
  * the CLI end to end with random weights, a ragged last batch, and with --compute_metrics.
"""
import json
import os

import numpy as np
import pytest
import torch

from kernel_check import rel_l2

pytestmark = pytest.mark.gpu

FORMS = {"nonlinear_k3": dict(kernel_size=3, padding=1, type="nonlinear"), "nonlinear_k1": dict(kernel_size=1, padding=0, type="nonlinear"),
         "linear": dict(kernel_size=3, padding=1, type="linear")}


def _cpu_rule(x):
    return x.add(1).div(2).mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8)


def _boundary_values():
    """Every fp32 value within 64 ulps of each x where save_image's rule steps from byte k-1 to k: (x + 1) / 2 * 255 + 0.5 = k."""
    k = torch.arange(1, 257, dtype=torch.float64)
    c = ((k - 0.5) / 255 * 2 - 1).float()
    vals, up, dn = [c], c.clone(), c.clone()
    for _ in range(64):
        up, dn = torch.nextafter(up, torch.tensor(np.inf)), torch.nextafter(dn, torch.tensor(-np.inf))
        vals += [up, dn]
    return torch.cat(vals)


def _run_save(vals, cuda, w=64):
    """vals fp32 [N] -> (device uint8 of N values, bytes past the output) through an NHWC [1, rows, w, 4] input whose pad channel is NaN."""
    from ladi_vton_b200 import lib, ops
    n = vals.numel()
    rows = -(-n // (3 * w))
    x = torch.full((1, rows, w, 4), float("nan"), dtype=torch.float32)
    flat = torch.zeros(rows * w * 3)
    flat[:n] = vals
    x[..., :3] = flat.view(1, rows, w, 3)
    x = x.to(cuda)
    guard = 4096
    buf = torch.full((rows * w * 3 + guard,), 0xA5, dtype=torch.uint8, device=cuda)
    lib.call("ladi_image_save_u8", ops._ptr(x), 1, rows, w, 4, ops._ptr(buf), ops._stream())
    torch.cuda.synchronize()
    out = buf[:rows * w * 3]
    assert torch.equal(out.view(1, rows, w, 3), ops.image_save_u8(x))  # the wrapper launches the same thing
    return out[:n].cpu(), buf[rows * w * 3:].cpu()


def test_image_save_u8_bit_exact(cuda):
    g = torch.Generator().manual_seed(0)
    special = torch.tensor([1.0, -1.0, np.inf, -np.inf, 2.0, -2.0, 1e30, -1e30, 1.0000001, -1.0000001, 0.0, -0.0, 3.4e38, -3.4e38,
                            1e-45, -1e-45])
    vals = torch.cat([_boundary_values(), torch.rand(1_000_000, generator=g) * 2.4 - 1.2, special])
    out, tail = _run_save(vals, cuda)
    ref = _cpu_rule(vals)
    bad = (out != ref).nonzero().flatten()
    assert bad.numel() == 0, [(float(vals[i]), int(out[i]), int(ref[i])) for i in bad[:10]]
    assert (tail == 0xA5).all(), "bytes past the output were written"
    out2, _ = _run_save(vals, cuda)
    assert torch.equal(out, out2)
    # every byte value is reached, and both rules are exercised at their steps
    assert set(out.tolist()) == set(range(256))
    assert out[-len(special):].tolist() == [255, 0, 255, 0, 255, 0, 255, 0, 255, 0, 128, 128, 255, 0, 128, 128]


def test_image_save_u8_nan(cuda):
    vals = torch.tensor([float("nan"), -float("nan"), 0.5, float("nan")])
    out, tail = _run_save(vals, cuda, w=2)
    assert out.tolist() == [0, 0, int(_cpu_rule(torch.tensor(0.5))), 0]
    assert (tail == 0xA5).all()


def _with_tf32_off(fn):
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        return fn()
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


def _engine_and_oracle(cuda, vae_cfg, vsd, esd, ein, eout, form):
    from ladi_oracle.emasc_forms import EMASC as OE
    from ladi_oracle.vae import AutoencoderKL as OV
    from ladi_vton_b200 import EMASC, AutoencoderKL
    vae = AutoencoderKL(**vae_cfg).load_state_dict(vsd).to(cuda)
    ov = OV(**vae_cfg).eval()
    ov.load_state_dict({k: v.cpu() for k, v in vsd.items()})
    em = oe = None
    if form != "none":
        kw = FORMS[form]
        em = EMASC(ein, eout, stride=1, **kw).load_state_dict(esd).to(cuda)
        oe = OE(ein, eout, **kw).eval()
        oe.load_state_dict({k: v.cpu() for k, v in esd.items()})
        oe = oe.to(cuda)
    return vae, em, ov.to(cuda), oe


def _recon(vae, em, ov, oe, batch, form, seed):
    """(engine decoded NHWC fp32 [B,H,W,3], engine uint8, oracle `(x + 1) / 2` NCHW fp32), each after seeding the CUDA RNG alike."""
    from ladi_oracle.vae_val_body import run_batch
    from ladi_vton_b200 import ops
    from ladi_vton_b200.eval import vae_recon_batch
    t = "none" if form == "none" else FORMS[form]["type"]
    torch.cuda.manual_seed(seed)
    img = vae_recon_batch(vae, em, batch, [1, 2, 3, 4, 5], t)
    u8 = ops.image_save_u8(img)
    odev = next(ov.parameters()).device
    dev = {k: (v.to(odev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    torch.cuda.manual_seed(seed)
    ref = _with_tf32_off(lambda: run_batch(dev, ov, oe, [1, 2, 3, 4, 5], t))
    return img[..., :3], u8, ref


@pytest.mark.parametrize("form", ["nonlinear_k3", "nonlinear_k1", "linear", "none"])
def test_reconstruction_small(cuda, form):
    import importlib.util
    spec = importlib.util.spec_from_file_location("g", os.path.join(os.path.dirname(__file__), "golden", "make_emasc_val_golden.py"))
    G = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(G)
    from ladi_vton_b200 import synthetic as S
    vsd, esd, (ein, eout) = G.state_dicts()
    vae, em, ov, oe = _engine_and_oracle(cuda, S.SMALL_VAE, vsd, esd.get(form if form != "none" else "nonlinear_k3"), ein, eout, form)
    with torch.no_grad():
        img, u8, ref = _recon(vae, em, ov, oe, G.inputs(), form, 77)
    dec_ref = (ref * 2 - 1).permute(0, 2, 3, 1)
    err, mad = rel_l2(img, dec_ref), float((img - dec_ref).abs().mean())
    print(f"\n[emasc val small {form}] decoded rel-L2 {err:.4f}, mean |d| {mad:.4f}")
    assert u8.shape == (2, G.H, G.W, 3)
    assert err < 5e-2 and mad < 2e-2


def test_reconstruction_full_size_batch16(cuda):
    """The trainer's shape: batch 16 (--test_batch_size), 512x384, full VAE and the hub's nonlinear 3x3 EMASC, random weights."""
    from ladi_oracle.vae_val_body import save_image_u8
    from ladi_vton_b200 import synthetic as S
    from ladi_vton_b200.eval import EMASC_IN, EMASC_OUT
    from ladi_vton_b200.vae import vae_param_shapes
    vsd = S.random_state_dict(vae_param_shapes({}), 1235, device=cuda, fast=True)
    esd = S.random_state_dict(S.emasc_param_shapes(EMASC_IN, EMASC_OUT), 1236, device=cuda, fast=True)
    vae, em, ov, oe = _engine_and_oracle(cuda, {}, vsd, esd, EMASC_IN, EMASC_OUT, "nonlinear_k3")
    inp = S.synthetic_inputs(16, 512, 384, seed=9, ctx_dim=8)
    mask = (inp["mask_image"] >= 0.5).float()
    batch = dict(image=inp["image"], im_mask=inp["image"] * (1 - mask), inpaint_mask=mask)
    with torch.no_grad():
        img, u8, ref = _recon(vae, em, ov, oe, batch, "nonlinear_k3", 5)
        ref_u8 = save_image_u8(ref)
    dec_ref = (ref * 2 - 1).permute(0, 2, 3, 1)
    errs = [rel_l2(img[i], dec_ref[i]) for i in range(16)]
    mads = [float((u8[i].float() - ref_u8[i].float()).abs().mean()) / 255 for i in range(16)]
    print(f"\n[emasc val 16x512x384] per-image decoded rel-L2 {min(errs):.4f}..{max(errs):.4f} (first {errs[0]:.4f}, last {errs[-1]:.4f}); "
          f"uint8 mean |d| {min(mads) * 255:.3f}..{max(mads) * 255:.3f} /255")
    assert max(errs) < 5e-2
    assert max(mads) <= 2 / 255


def _gt_tree(root, n):
    """The VITON-HD test tree compute_metrics reads the ground truth from: test_pairs.txt and test/image/<name>."""
    from PIL import Image
    rs = np.random.RandomState(15)
    names = [f"{i:05d}_00.jpg" for i in range(n)]
    os.makedirs(os.path.join(root, "test", "image"))
    with open(os.path.join(root, "test_pairs.txt"), "w") as f:
        f.write("".join(f"{a} {a}\n" for a in names))
    for nm in names:
        Image.fromarray(rs.randint(0, 256, size=(8, 6, 3)).astype(np.uint8)).resize((384, 512)).save(os.path.join(root, "test", "image", nm))


def test_cli_end_to_end(cuda, tmp_path, monkeypatch):
    """--random_init --synthetic_samples 20 --test_batch_size 16 (a ragged last batch of 4): the reference's tree and names, JPEG files,
    byte-identical files from two runs with the same seed, and with --compute_metrics the metrics JSON."""
    from PIL import Image
    from ladi_vton_b200.eval_emasc import main
    monkeypatch.setenv("HOME", str(tmp_path))  # the ground-truth statistics cache (~/.cache/ladi_vton_b200/metrics)
    root = str(tmp_path / "vitonhd")
    _gt_tree(root, 20)
    argv = ["--dataset", "vitonhd", "--vitonhd_dataroot", root, "--synthetic_samples", "20", "--test_batch_size", "16", "--random_init"]
    w1 = main(argv + ["--output_dir", str(tmp_path / "a")])
    w2 = main(argv + ["--output_dir", str(tmp_path / "b"), "--compute_metrics"])
    names = [f"{i:05d}_00.jpg" for i in range(20)]
    d = tmp_path / "a" / "imgs_step_random_init_paired" / "upper_body"
    assert sorted(os.listdir(d)) == names and w1 == [str(d / n) for n in names]
    assert sorted(os.listdir(tmp_path / "a")) == ["imgs_step_random_init_paired"]
    for p in w1:
        raw = open(p, "rb").read()
        assert raw[:3] == b"\xff\xd8\xff"
        im = Image.open(p)
        assert im.format == "JPEG" and im.size == (384, 512) and im.mode == "RGB"
    for a, b in zip(w1, w2):
        assert open(a, "rb").read() == open(b, "rb").read(), (a, b)
    out = json.load(open(tmp_path / "b" / "metrics_imgs_step_random_init_paired_all.json"))
    assert list(out) == ['ssim_score', 'lpips_score', 'fid_score', 'kid_score', 'is_score'], out
    assert all(np.isfinite(v) for v in out.values()), out
    print(f"\n[emasc validation] metrics: {out}")
