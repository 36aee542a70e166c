"""Host-side tests of the image-quality metrics (ladi_vton_b200/metrics.py, ladi_vton_b200/val_metrics.py) and of their oracle
(oracle/ladi_oracle/metrics.py): the oracle networks against torchvision's Inception-v3 (with the FID pool variants) and AlexNet, the
weight packing (BatchNorm fold, (ky, kx, c) im2col columns) against F.conv2d, closed forms of the statistics, and the CLI (flags against
the reference parser, error texts, folder listing and name matching).  No GPU needed."""
import json
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "metrics_flags.json")))


# ---- networks -------------------------------------------------------------------------------------------------------------------------
def _fid_torchvision():
    """torchvision inception_v3(1008 classes, no aux logits) with the FID blocks' pools: count_include_pad=False in A, C and E_1, a 3x3
    max pool in E_2 (pytorch-fid's FIDInceptionA / C / E_1 / E_2)."""
    import torchvision
    net = torchvision.models.inception_v3(weights=None, num_classes=1008, aux_logits=False, init_weights=False).eval()

    def a(self, x):
        return [self.branch1x1(x), self.branch5x5_2(self.branch5x5_1(x)),
                self.branch3x3dbl_3(self.branch3x3dbl_2(self.branch3x3dbl_1(x))),
                self.branch_pool(F.avg_pool2d(x, 3, 1, 1, count_include_pad=False))]

    def c(self, x):
        b7 = self.branch7x7_3(self.branch7x7_2(self.branch7x7_1(x)))
        bd = self.branch7x7dbl_5(self.branch7x7dbl_4(self.branch7x7dbl_3(self.branch7x7dbl_2(self.branch7x7dbl_1(x)))))
        return [self.branch1x1(x), b7, bd, self.branch_pool(F.avg_pool2d(x, 3, 1, 1, count_include_pad=False))]

    def e(pool):
        def fwd(self, x):
            t = self.branch3x3_1(x)
            b3 = torch.cat([self.branch3x3_2a(t), self.branch3x3_2b(t)], 1)
            t = self.branch3x3dbl_2(self.branch3x3dbl_1(x))
            bd = torch.cat([self.branch3x3dbl_3a(t), self.branch3x3dbl_3b(t)], 1)
            return [self.branch1x1(x), b3, bd, self.branch_pool(pool(x))]
        return fwd

    for m in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
        getattr(net, m)._forward = types.MethodType(a, getattr(net, m))
    for m in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
        getattr(net, m)._forward = types.MethodType(c, getattr(net, m))
    net.Mixed_7b._forward = types.MethodType(e(lambda x: F.avg_pool2d(x, 3, 1, 1, count_include_pad=False)), net.Mixed_7b)
    net.Mixed_7c._forward = types.MethodType(e(lambda x: F.max_pool2d(x, 3, 1, 1)), net.Mixed_7c)
    return net


def test_inception_state_dict_layout():
    """Key set and shapes equal torchvision's: a real pt_inception-2015-12-05 file loads strictly."""
    from ladi_vton_b200.metrics import FIDInceptionV3
    ref = {k: tuple(v.shape) for k, v in _fid_torchvision().state_dict().items()}
    assert FIDInceptionV3().param_shapes() == ref


def test_oracle_inception_matches_torchvision():
    from ladi_oracle import metrics as OM
    torch.manual_seed(0)
    net = _fid_torchvision()
    with torch.no_grad():
        for m in net.modules():  # non-trivial BatchNorm statistics
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.uniform_(-0.1, 0.1), m.running_var.uniform_(0.5, 1.5), m.weight.uniform_(0.5, 1.5), m.bias.uniform_(-0.1, 0.1)
    sd = net.state_dict()
    x = torch.rand(2, 3, 139, 139) * 255
    seen = {}
    net.fc.register_forward_hook(lambda mod, inp, out: seen.update(f=inp[0], logits=out))
    with torch.no_grad():
        net((x - 128) / 128)
        f, logits = OM.inception_features(sd, x)
    assert torch.equal(f, seen["f"])
    assert torch.allclose(logits, (seen["logits"] - sd["fc.bias"]).double(), rtol=1e-5, atol=1e-5)


def test_oracle_alexnet_taps_bit_exact():
    import torchvision
    from ladi_oracle import metrics as OM
    torch.manual_seed(1)
    feats = torchvision.models.alexnet(weights=None).features.eval()
    sd = {f"features.{k}": v for k, v in feats.state_dict().items()}
    x = torch.randn(2, 3, 131, 99)
    with torch.no_grad():
        taps = OM.alexnet_taps(sd, x)
        ref, y = [], x
        for lo, hi in ((0, 2), (2, 5), (5, 8), (8, 10), (10, 12)):  # lpips.pretrained_networks.alexnet slices
            y = feats[lo:hi](y)
            ref.append(y)
    for a, b in zip(taps, ref):
        assert torch.equal(a, b)
    from ladi_vton_b200.metrics import LPIPSAlex
    shapes = LPIPSAlex().param_shapes()
    assert {k: v for k, v in shapes.items() if k.startswith("features.")} == {k: tuple(v.shape) for k, v in sd.items()}
    assert [shapes[f"lin{i}.model.1.weight"][1] for i in range(5)] == [t.shape[1] for t in taps]


def _im2col_rows(x_nchw, kernel, stride, padding, k_pad):
    """What ladi_im2col_bf16 writes, restated with torch: rows (n, oy, ox), columns (ky, kx, c), zeros beyond kh*kw*c."""
    (kh, kw), (sh, sw), (ph, pw) = kernel, stride, padding
    xp = F.pad(x_nchw, (pw, pw, ph, ph))
    n, c = x_nchw.shape[:2]
    oh, ow = (xp.shape[2] - kh) // sh + 1, (xp.shape[3] - kw) // sw + 1
    cols = [xp[:, :, ky:ky + sh * (oh - 1) + 1:sh, kx:kx + sw * (ow - 1) + 1:sw] for ky in range(kh) for kx in range(kw)]
    rows = torch.stack(cols, 1).permute(0, 3, 4, 1, 2).reshape(n * oh * ow, kh * kw * c)
    return F.pad(rows, (0, k_pad - rows.shape[1])), (n, oh, ow)


@pytest.mark.parametrize("kernel,stride,padding,ci", [((1, 7), (1, 1), (0, 3), 16), ((7, 1), (1, 1), (3, 0), 16), ((5, 5), (1, 1), (2, 2), 8),
                                                     ((11, 11), (4, 4), (2, 2), 3), ((3, 3), (2, 2), (0, 0), 24), ((3, 3), (1, 1), (0, 0), 32),
                                                     ((1, 3), (1, 1), (0, 1), 8), ((3, 1), (1, 1), (1, 0), 8)])
def test_bn_fold_and_im2col_layout(kernel, stride, padding, ci):
    from ladi_vton_b200.metrics import fold_bn, pack_im2col_weight
    from ladi_vton_b200.weights import pad64
    g = torch.Generator().manual_seed(3)
    co = 24
    w = torch.randn(co, ci, *kernel, generator=g, dtype=torch.float64)
    gamma, beta = torch.rand(co, generator=g, dtype=torch.float64) + 0.5, torch.randn(co, generator=g, dtype=torch.float64)
    mean, var = torch.randn(co, generator=g, dtype=torch.float64), torch.rand(co, generator=g, dtype=torch.float64) + 0.5
    x = torch.randn(2, ci, 23, 19, generator=g, dtype=torch.float64)
    ref = F.batch_norm(F.conv2d(x, w, None, stride, padding), mean, var, gamma, beta, False, 0.0, 1e-3)
    wf, bf = fold_bn(w, gamma, beta, mean, var, 1e-3)
    assert torch.allclose(F.conv2d(x, wf, None, stride, padding) + bf.view(1, -1, 1, 1), ref, atol=1e-10)
    packed = pack_im2col_weight(wf)
    assert packed.dtype == torch.bfloat16 and packed.shape == (co, pad64(kernel[0] * kernel[1] * ci))
    rows, (n, oh, ow) = _im2col_rows(x, kernel, stride, padding, packed.shape[1])
    got = (rows @ packed.double().T).view(n, oh, ow, co).permute(0, 3, 1, 2)
    want = F.conv2d(x, wf.to(torch.bfloat16).double(), None, stride, padding)
    assert torch.allclose(got, want, atol=1e-10)


def test_implicit_3x3_rule():
    from ladi_vton_b200.metrics import INCEPTION_LAYERS, uses_implicit_3x3
    assert uses_implicit_3x3((3, 3), (1, 1), (1, 1), 8) and not uses_implicit_3x3((3, 3), (1, 1), (1, 1), 35)
    assert not uses_implicit_3x3((3, 3), (2, 2), (0, 0), 8) and not uses_implicit_3x3((1, 7), (1, 1), (0, 3), 8)
    # every channel count is a multiple of 8 (branch outputs land in concat slices at 16-byte aligned offsets)
    assert all(ci % 8 == 0 or ci == 3 for ci, *_ in INCEPTION_LAYERS.values()) and all(co % 8 == 0 for _, co, *_ in INCEPTION_LAYERS.values())


# ---- closed forms -------------------------------------------------------------------------------------------------------------------
def test_ssim_oracle_closed_forms():
    from ladi_oracle import metrics as OM
    x = torch.rand(3, 3, 40, 31, generator=torch.Generator().manual_seed(4))
    assert torch.allclose(OM.ssim(x, x), torch.ones(3, dtype=torch.float64), atol=1e-12)
    a, b = 0.3, 0.7
    s = OM.ssim(torch.full((1, 3, 20, 20), a), torch.full((1, 3, 20, 20), b))
    c1 = 0.01 ** 2
    assert abs(float(s[0]) - (2 * a * b + c1) / (a * a + b * b + c1)) < 1e-7


def test_frechet_distance_diagonal():
    from ladi_vton_b200.metrics import frechet_distance
    g = np.random.RandomState(5)
    mu1, mu2 = g.randn(6), g.randn(6)
    s1, s2 = g.rand(6) + 0.1, g.rand(6) + 0.1
    want = ((mu1 - mu2) ** 2).sum() + (s1 + s2 - 2 * np.sqrt(s1 * s2)).sum()
    assert abs(frechet_distance(mu1, np.diag(s1), mu2, np.diag(s2)) - want) < 1e-9
    assert abs(frechet_distance(mu1, np.diag(s1), mu1, np.diag(s1))) < 1e-9


def test_frechet_distance_singular_product_retries():
    from ladi_vton_b200.metrics import frechet_distance
    s = np.zeros((4, 4))
    s[0, 0] = 1.0  # rank-deficient covariances
    assert np.isfinite(frechet_distance(np.zeros(4), s, np.ones(4), s))


def test_kernel_distance_matches_double_loop():
    from ladi_oracle import metrics as OM
    from ladi_vton_b200.metrics import kernel_distance
    g = np.random.RandomState(6)
    f1, f2 = g.randn(14, 5), g.randn(11, 5) + 0.3
    for seed in (0, 9):
        a = kernel_distance(f1, f2, num_subsets=4, max_subset_size=8, seed=seed)
        b = OM.kernel_distance_direct(f1, f2, num_subsets=4, max_subset_size=8, seed=seed)
        assert abs(a - b) < 1e-10 * max(1.0, abs(b))
    assert kernel_distance(f1, f2, num_subsets=4, seed=2) == kernel_distance(f1, f2, num_subsets=4, seed=2)


def test_inception_score_closed_forms():
    from ladi_oracle import metrics as OM
    from ladi_vton_b200.metrics import inception_score
    assert abs(inception_score(np.zeros((40, 1008)))[0] - 1.0) < 1e-12
    k = 7
    onehot = np.full((k * 5, 1008), -40.0)  # exp(-40) * 1007 ~ 4e-15 off-class mass
    onehot[np.arange(k * 5), np.arange(k * 5) % k] = 0.0
    assert abs(inception_score(onehot, splits=1)[0] - k) < 1e-9
    z = np.random.RandomState(7).randn(23, 1008) * 3  # ragged chunks (torch.chunk: 3 rows each, 8 chunks)
    for seed in (0, 4):
        m, s = inception_score(z, seed=seed)
        om, os_ = OM.inception_score(z, seed=seed)
        assert abs(m - om) < 1e-12 and abs(s - os_) < 1e-12


def test_clean_resize_matches_oracle():
    from ladi_oracle import metrics as OM
    from ladi_vton_b200.val_metrics import clean_resize
    img = (np.random.RandomState(8).rand(64, 48, 3) * 255).astype(np.uint8)
    out = clean_resize(img)
    assert out.shape == (299, 299, 3) and out.dtype == np.float32 and out.min() >= 0 and out.max() <= 255
    assert np.array_equal(out, OM.clean_resize(img))


# ---- CLI ------------------------------------------------------------------------------------------------------------------------------
def test_flags_match_reference_parser():
    from ladi_vton_b200.val_metrics import build_parser
    parser = build_parser()
    acts = {a.option_strings[0]: a for a in parser._actions if a.option_strings and a.option_strings[0] != "-h"}
    engine = {a.option_strings[0] for g in parser._action_groups if g.title == "engine" for a in g._group_actions}
    assert engine == {"--metrics_weights_dir", "--cache_dir", "--random_init", "--seed"}
    ref_names = [f["flags"][0] for f in GOLD["flags"]]
    assert len(ref_names) == 8
    assert sorted(set(acts) - engine) == sorted(ref_names)
    for f in GOLD["flags"]:
        a = acts[f["flags"][0]]
        assert a.option_strings == f["flags"]
        assert a.type.__name__ == f["type"], f
        assert a.default == f.get("default"), f
        assert bool(a.required) == bool(f.get("required", False)), f
        assert (list(a.choices) if a.choices else None) == f.get("choices"), f


def test_reference_errors(tmp_path):
    from ladi_vton_b200.val_metrics import build_parser, check_args, main
    base = ["--gen_folder", str(tmp_path), "--test_order", "paired"]
    with pytest.raises(ValueError, match="VitonHD dataroot must be provided"):
        check_args(build_parser().parse_args(base + ["--dataset", "vitonhd"]))
    with pytest.raises(ValueError, match="DressCode dataroot must be provided"):
        check_args(build_parser().parse_args(base + ["--dataset", "dresscode"]))
    with pytest.raises(ValueError, match="The generated images folder does not exist"):
        check_args(build_parser().parse_args(["--gen_folder", str(tmp_path / "nope"), "--test_order", "paired", "--dataset", "vitonhd",
                                              "--vitonhd_dataroot", "/d"]))
    (tmp_path / "w").mkdir()
    (tmp_path / "w" / "alex.pth").write_bytes(b"")
    with pytest.raises(FileNotFoundError, match="pt_inception-2015-12-05-6726825d.pth, alexnet-owt-7be5be79.pth") as e:
        main(base + ["--dataset", "vitonhd", "--vitonhd_dataroot", "/d", "--metrics_weights_dir", str(tmp_path / "w")])
    assert "alex.pth," not in str(e.value)
    with pytest.raises(FileNotFoundError, match="alex.pth"):
        main(base + ["--dataset", "vitonhd", "--vitonhd_dataroot", "/d"])


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only check")
def test_no_cpu_path(tmp_path):
    from ladi_vton_b200.metrics import FIDInceptionV3
    from ladi_vton_b200.val_metrics import main
    with pytest.raises(RuntimeError, match="no CPU path"):
        FIDInceptionV3().to("cpu")
    with pytest.raises(RuntimeError, match="no CPU path"):
        main(["--gen_folder", str(tmp_path), "--test_order", "paired", "--dataset", "vitonhd", "--vitonhd_dataroot", "/d", "--random_init"])
    assert os.listdir(tmp_path) == []


def _touch(path):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    open(path, "wb").close()


def test_vitonhd_listing_and_stats(tmp_path):
    from ladi_vton_b200.val_metrics import custom_stats_paths, folder_images, gen_paths, gt_paths
    root, gen = str(tmp_path / "vitonhd"), str(tmp_path / "gen")
    names = ["00017_00.jpg", "00006_00.jpg", "00034_00.jpg"]
    os.makedirs(root)
    with open(os.path.join(root, "test_pairs.txt"), "w") as f:
        f.write("".join(f"{n} {c}\n" for n, c in zip(names, reversed(names))))
    for n in names + ["99999_00.jpg"]:
        _touch(os.path.join(root, "test", "image", n))
    for n in names:
        _touch(os.path.join(gen, "upper_body", n.replace(".jpg", ".png")))
    want_gt = [os.path.join(root, "test", "image", n) for n in sorted(names)]
    assert gt_paths(root, "vitonhd", "all") == want_gt == gt_paths(root, "vitonhd", "upper_body")
    g = gen_paths(gen, "all")
    assert [os.path.splitext(os.path.basename(p))[0] for p in g] == [os.path.splitext(os.path.basename(p))[0] for p in want_gt]
    assert gen_paths(gen, "upper_body") == g
    # the statistics use the whole test/image folder, for 'all' and 'upper_body' alike
    assert custom_stats_paths("vitonhd", "all", None, root) == folder_images(os.path.join(root, "test", "image"))
    assert len(custom_stats_paths("vitonhd", "upper_body", None, root)) == 4
    with pytest.raises(ValueError, match="vitonhd_lower_body"):
        custom_stats_paths("vitonhd", "lower_body", None, root)
    with open(os.path.join(gen, "metrics_paired_all.json"), "w") as f:
        f.write("{}")
    assert folder_images(gen) == g  # json results next to the images are not images


def test_dresscode_listing_per_category(tmp_path):
    from ladi_vton_b200.val_metrics import custom_stats_paths, gen_paths, gt_paths
    root, gen = str(tmp_path / "dc"), str(tmp_path / "gen")
    per_cat = {"upper_body": ["000010_0.jpg", "000002_0.jpg"], "lower_body": ["013563_0.jpg"], "dresses": ["020714_0.jpg", "020700_0.jpg"]}
    lines = [n for c in ("dresses", "upper_body", "lower_body") for n in per_cat[c]] + ["055555_0.jpg"]  # one line has no image
    os.makedirs(root)
    with open(os.path.join(root, "test_pairs_paired.txt"), "w") as f:
        f.write("".join(f"{n} {n.replace('_0', '_1')}\n" for n in lines))
    for c, ns in per_cat.items():
        for n in ns:
            _touch(os.path.join(root, c, "images", n))
            _touch(os.path.join(gen, c, n))
    for c, ns in per_cat.items():
        assert gt_paths(root, "dresscode", c) == sorted(os.path.join(root, c, "images", n) for n in ns)
        assert [os.path.basename(p) for p in gen_paths(gen, c)] == sorted(ns)
        assert custom_stats_paths("dresscode", c, root, None) == sorted(os.path.join(root, c, "images", n) for n in ns)
    gt_all, gen_all = gt_paths(root, "dresscode", "all"), gen_paths(gen, "all")
    assert len(gt_all) == len(gen_all) == 5
    # GTTestDataset sorts full paths (category folder first) and GenTestDataset likewise: the pairs line up by name
    assert [os.path.basename(p) for p in gt_all] == [os.path.basename(p) for p in gen_all]
    assert [os.path.basename(p) for p in custom_stats_paths("dresscode", "all", root, None)] == sorted(n for ns in per_cat.values() for n in ns)
    with pytest.raises(ValueError, match="DressCode dataroot must be provided"):
        custom_stats_paths("dresscode", "all", None, None)
