"""The wgmma attention kernels at the edges of their schedules and under the score distributions online softmax gets wrong, against float64.

`attention_d64_kernel` (`ladi_attention_bf16`, every UNet attn1 / attn2) is persistent: grid_x = min(items, SMs) CTAs, an item is one
(192-row query tile, head, image), numbered query tile fastest, and CTA c runs items c, c + grid_x, ...  Its Q tile is double-buffered
across items (item `it` of a CTA uses buffer it & 1 at phase (it >> 1) & 1, so the phase first returns at the fifth item), K and V go
through a 4-stage ring whose tile counter carries from one item into the next, and its three consumer warpgroups take turns issuing
MMAs through named barriers, a turn order that also carries across items (an item takes n_kv_tiles + 1 turns).
`attention_kernel<D>` (`ladi_attention_d512_bf16`, D = 512 / 256) runs one CTA per (128-row query tile, 128-column output slice, image)
over 64-key tiles.  `ladi_attention_plan` reports what either launch runs; it shares the validation-and-policy function with the launches
and needs no device.

The GPU cases reach: item counts of 1, sms - 1, sms, sms + 1, 2 sms + 1, 4 sms + 1 and 8 sms + 3 (up to 9 items per CTA, so the Q
buffer phase wraps twice); 1, 2, 3, 4, 5, 8 and 9 key tiles per item at >= 5 items per CTA, so that between them items start at every
ring stage and phase and with every warpgroup holding the turn; query tails nq mod 192 of 1, 64, 65, 128, 129 and 191 at >= 3 items per
CTA (0, 1 or 2 idle consumer warpgroups in every CTA's last query tiles); every score distribution of tests/kernel_check.py (randn, late,
early, tail, flat, level) at one and at many items per CTA and through the fused-QKV placement; the late maximum over 96 key tiles
(12288 keys, the 1024x768 level-0 length); and the wide kernel under every distribution.  Each case first asserts its plan at the
device's SM count (the launch runs the grid the plan names), then is checked the way the workload census checks the workload's calls:
against float64 with the per-element bound `attn_expect`, bit for bit against a second run, and with every byte of the output buffer
outside the rows and columns the call owns (pitch gaps, the gap between batch images) NaN-poisoned before the call and still NaN after
it.  Every input pitch gap and batch gap is NaN too.  Each case prints its plan and its worst err/bound.

The CPU tests pin the plan tables (every attention descriptor of the workload census and every GPU case, at 132 SMs) and show that the
bound has teeth: an fp32 emulation of the kernels' online softmax (`emulate_attn`) passes on every distribution at 128- and 64-key tiles,
and each simulated fault is rejected on the distribution built to expose it."""
import ctypes as C

import pytest
import torch

from kernel_check import (ATTN_DISTS, SMS, Replay, addr, attn_expect, attn_inputs, attn_ref, census, emulate_attn, ladi_lib, max_ratio,
                          plan_query, ratio, same, sms)

SCALE = 0.125
PAD = 24  # columns of NaN after each row of every operand (keeps the pitch a multiple of 8)
GAP = 40  # NaN elements between consecutive batch images
PLAN_FIELDS = ("head_dim", "grid_x", "grid_y", "grid_z", "q_tile", "kv_tile", "stages", "consumers", "n_q_tiles", "n_kv_tiles", "n_items",
               "items_min", "items_max", "idle_consumers_last_q_tile", "smem_bytes")
SMEM = {64: 2 * 192 * 128 + 2 * 4 * 128 * 128 + (4 + 16) * 8 + 1024, 512: 8 * 128 * 128 + 10 * 64 * 128 + 21 * 8 + 1024,
        256: 4 * 128 * 128 + 10 * 64 * 128 + 21 * 8 + 1024}


# ================================================================================================================ plans
def cdiv(a, b):
    return -(-a // b)


def expected_plan(B, heads, nq, nkv, D, n_sms):
    """The launch policy restated: D = 64 192-row query tiles, 128-key tiles, 4 stages, 3 consumers, persistent over min(items, SMs)
    CTAs; D = 512 / 256 128-row query tiles, 64-key tiles, a 10-chunk ring, 2 consumers, one CTA per (query tile, 128-column slice,
    image)."""
    qt, kt, stages, cons = (192, 128, 4, 3) if D == 64 else (128, 64, 10, 2)
    nqt, nkt = cdiv(nq, qt), cdiv(nkv, kt)
    idle = cons - cdiv(nq - (nqt - 1) * qt, 64)
    if D == 64:
        items = nqt * heads * B
        grid = (min(items, n_sms), 1, 1)
        per = (items // grid[0], cdiv(items, grid[0]))
    else:
        grid = (nqt, D // 128, B)
        items, per = nqt * D // 128 * B, (1, 1)
    return dict(head_dim=D, grid_x=grid[0], grid_y=grid[1], grid_z=grid[2], q_tile=qt, kv_tile=kt, stages=stages, consumers=cons,
                n_q_tiles=nqt, n_kv_tiles=nkt, n_items=items, items_min=per[0], items_max=per[1], idle_consumers_last_q_tile=idle,
                smem_bytes=SMEM[D])


def attn_desc(B, heads, nq, nkv, D=64, **kw):
    """A dense descriptor on fake 256-byte aligned addresses (the plan query dereferences nothing); kw overrides fields."""
    d = ladi_lib().AttnDesc()
    W = heads * D
    d.batch, d.heads, d.nq, d.nkv, d.scale, d.head_dim = B, heads, nq, nkv, SCALE if D == 64 else D ** -0.5, 0 if D == 64 else D
    d.q, d.q_pitch, d.q_batch_stride = addr(1), W, nq * W
    d.k, d.k_pitch, d.k_batch_stride = addr(2), W, nkv * W
    d.v, d.v_pitch, d.v_batch_stride = addr(3), W, nkv * W
    d.out, d.out_pitch, d.out_batch_stride = addr(4), W, nq * W
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def plan_of(d, wide, n_sms):
    """-> (plan dict, "") or (None, error message)."""
    return plan_query("ladi_attention_plan", ladi_lib().AttnPlan, [C.byref(d), 1 if wide else 0, n_sms], PLAN_FIELDS)


# ================================================================================================================ the GPU cases
# Each case: (B, heads, nq, nkv, dist, fused, D, plan fields it targets) as a function of the SM count.
ITEMS = {"1": lambda s: 1, "sms-1": lambda s: s - 1, "sms": lambda s: s, "sms+1": lambda s: s + 1, "2sms+1": lambda s: 2 * s + 1,
         "4sms+1": lambda s: 4 * s + 1, "8sms+3": lambda s: 8 * s + 3}
ITEM_TAILS = {"1": 100, "sms-1": 1, "sms": 64, "sms+1": 129, "2sms+1": 191, "4sms+1": 65, "8sms+3": 128}  # nq mod 192 of the last tile


def items_case(label, s):
    n = ITEMS[label](s)  # one head, one image: the items are the query tiles
    return dict(B=1, heads=1, nq=192 * (n - 1) + ITEM_TAILS[label], nkv=200, want=dict(n_items=n, grid_x=min(n, s), items_max=cdiv(n, s)))


N_TILES = [1, 2, 3, 4, 5, 8, 9]


def ring_case(n_tiles, s):
    T = cdiv(5 * s, 8) + 1  # 8 (head, image) pairs: >= 5 items per CTA
    return dict(B=2, heads=4, nq=192 * (T - 1) + 150, nkv=128 * n_tiles - (37 if n_tiles % 2 else 0),
                want=dict(n_kv_tiles=n_tiles, items_min=5 if s == SMS else None))


TAIL_IDLE = {1: 2, 64: 2, 65: 1, 128: 1, 129: 0, 191: 0}


def tail_case(r, s):
    T = cdiv(3 * s, 6) + 1  # 6 (head, image) pairs: >= 3 items per CTA
    return dict(B=2, heads=3, nq=192 * (T - 1) + r, nkv=300, want=dict(idle_consumers_last_q_tile=TAIL_IDLE[r], items_min=3 if s == SMS else None))


DIST_NKV = {"randn": 300, "late": 128 * 5 - 20, "early": 300, "tail": 333, "flat": 45, "level": 300}  # tail / flat: ragged last tile
PLACEMENTS = ["one item", "many items", "fused"]


def dist_case(dist, placement, s):
    nkv = DIST_NKV[dist]
    if placement == "one item":
        return dict(B=2, heads=2, nq=300, nkv=nkv, want=dict(n_items=8, items_max=1))
    if placement == "many items":
        T = cdiv(4 * s, 12) + 1  # 12 (head, image) pairs: >= 4 items per CTA
        return dict(B=3, heads=4, nq=192 * (T - 1) + 77, nkv=nkv, want=dict(items_min=4 if s == SMS else None))
    return dict(B=2, heads=3, nq=nkv, nkv=nkv, fused=True, want=dict(n_q_tiles=cdiv(nkv, 192)))


WIDE_DIST_NKV = {"late": 64 * 7 + 10, "early": 300, "tail": 64 * 7 + 10, "flat": 45, "level": 300}


def all_cases(s):
    """Every parametrised GPU case of this file at `s` SMs: (id, case)."""
    out = [(f"items {k}", items_case(k, s)) for k in ITEMS]
    out += [(f"ring {n} tiles", ring_case(n, s)) for n in N_TILES]
    out += [(f"query tail {r}", tail_case(r, s)) for r in TAIL_IDLE]
    out += [(f"{dist} {p}", dict(dist_case(dist, p, s), dist=dist)) for dist in ATTN_DISTS for p in PLACEMENTS]
    out += [("late 96 tiles", dict(B=1, heads=2, nq=400, nkv=12288, dist="late", want=dict(n_kv_tiles=96)))]
    out += [(f"wide {D} {dist}", dict(B=3, heads=1, nq=200, nkv=WIDE_DIST_NKV[dist], D=D, dist=dist, want={}))
            for D in (512, 256) for dist in WIDE_DIST_NKV]
    return out


def check_plan(d, case, n_sms):
    """The case's plan at n_sms: the restated policy, and the fields the case targets."""
    D = case.get("D", 64)
    p, err = plan_of(d, D != 64, n_sms)
    assert p is not None, err
    assert p == expected_plan(case["B"], case["heads"], case["nq"], case["nkv"], D, n_sms), p
    for k, v in case["want"].items():
        assert v is None or p[k] == v, (k, p[k], v)
    return p


def _place(buf, vals, pitch, bstride, col0=0):
    buf.as_strided(vals.shape, (bstride, pitch, 1), col0).copy_(vals)


def run_case(R, B, heads, nq, nkv, fused=False, D=64, dist="randn", want=None):
    """D = 64: ladi_attention_bf16 with `heads` heads; D = 512 / 256: ladi_attention_d512_bf16 (heads must be 1, head_dim = D).  Inputs
    from attn_inputs(dist); the plan is asserted at the device's SM count first.  -> the worst err/bound over the images."""
    lib = ladi_lib()
    width = heads * D
    scale = SCALE if D == 64 else D ** -0.5
    q, k, v = attn_inputs(dist, R.g, B, heads, nq, nkv, D, scale, 128 if D == 64 else 64)
    d = lib.AttnDesc()
    d.batch, d.heads, d.nq, d.nkv, d.scale, d.variant = B, heads, nq, nkv, scale, 0
    d.head_dim = 0 if D == 64 else D
    nan = lambda n: torch.full((n,), float("nan"), dtype=torch.bfloat16, device=R.dev)  # noqa: E731
    if fused:  # one [B][n][3 * width + PAD] projection output: q, k, v are column slices of it
        assert nq == nkv
        pitch = 3 * width + PAD
        bs = nq * pitch + GAP
        buf = nan((B - 1) * bs + nq * pitch)
        for i, t in enumerate((q, k, v)):
            _place(buf, t, pitch, bs, i * width)
        base = buf.data_ptr()
        d.q, d.k, d.v = base, base + 2 * width, base + 4 * width
        d.q_pitch = d.k_pitch = d.v_pitch = pitch
        d.q_batch_stride = d.k_batch_stride = d.v_batch_stride = bs
        keep = [buf]
    else:
        pitch = width + PAD
        keep = []
        for name, t, n in (("q", q, nq), ("k", k, nkv), ("v", v, nkv)):
            b_ = nan((B - 1) * (n * pitch + GAP) + n * pitch)
            _place(b_, t, pitch, n * pitch + GAP)
            setattr(d, name, b_.data_ptr())
            setattr(d, name + "_pitch", pitch)
            setattr(d, name + "_batch_stride", n * pitch + GAP)
            keep.append(b_)
    op, obs = width + PAD, nq * (width + PAD) + GAP
    d.out_pitch, d.out_batch_stride = op, obs
    outs = [nan((B - 1) * obs + nq * op) for _ in range(2)]
    d.out = outs[0].data_ptr()
    p = check_plan(d, dict(B=B, heads=heads, nq=nq, nkv=nkv, D=D, want=want or {}), sms(R.dev))
    for o in outs:
        d.out = o.data_ptr()
        lib.call("ladi_attention_bf16" if D == 64 else "ladi_attention_d512_bf16", C.byref(d), R.stream)
    torch.cuda.synchronize()
    del keep
    out = outs[0]
    owned = torch.zeros(out.shape, dtype=torch.bool, device=R.dev)
    owned.as_strided((B, nq, width), (obs, op, 1)).fill_(True)
    assert bool(torch.isfinite(out[owned].float()).all()), "unwritten or NaN-contaminated output element"
    assert bool(torch.isnan(out[~owned].float()).all()), "wrote outside its rows and columns (pitch gap or batch gap)"
    assert same(outs[0], outs[1]), "two runs differ bitwise"
    ov = out.as_strided((B, nq, width), (obs, op, 1))
    worst = 0.0
    for b in range(B):
        o64, sv = attn_ref(q[b].double(), k[b].double(), v[b].double(), heads, D, scale)
        w = max_ratio(ov[b], o64, attn_expect(o64, sv, nkv))
        assert w <= 1.0, f"image {b}: err/bound {w:.3g}"
        worst = max(worst, w)
    print(f"\nD={D} {dist}{' fused' if fused else ''} B={B} heads={heads} nq={nq} nkv={nkv}: {p['n_items']} items on {p['grid_x']}x"
          f"{p['grid_y']}x{p['grid_z']} CTAs ({p['items_min']}-{p['items_max']} per CTA), {p['n_kv_tiles']} key tiles, "
          f"{p['idle_consumers_last_q_tile']} idle consumers in the last query tile; worst err/bound {worst:.3g}")
    return worst


# ================================================================================================================ CPU: plan tables
def test_plan_constants():
    """192 / 128 / 4 stages / 3 consumers for D = 64; 128 / 64 / 10 / 2 for the wide kernel."""
    p, err = plan_of(attn_desc(2, 5, 3072, 3072), False, SMS)
    assert (p["q_tile"], p["kv_tile"], p["stages"], p["consumers"], p["smem_bytes"]) == (192, 128, 4, 3, 181408), err
    for D, smem in ((512, 214184), (256, 148648)):
        p, err = plan_of(attn_desc(1, 1, 3072, 3072, D=D), True, SMS)
        assert (p["q_tile"], p["kv_tile"], p["stages"], p["consumers"], p["smem_bytes"]) == (128, 64, 10, 2, smem), err


# (B, heads, nq, nkv, D) -> (grid_x, grid_y, grid_z, n_items, items_min, items_max, idle) at 132 SMs
PLAN_TABLE = [
    ("UNet level 0 attn1, 8 x 512x384 with CFG", (16, 5, 3072, 3072, 64), (132, 1, 1, 1280, 9, 10, 0)),
    ("UNet level 0 attn2", (16, 5, 3072, 77, 64), (132, 1, 1, 1280, 9, 10, 0)),
    ("UNet level 2 attn1", (16, 20, 192, 192, 64), (132, 1, 1, 320, 2, 3, 0)),
    ("UNet level 0 attn1, 1024x768", (2, 5, 12288, 12288, 64), (132, 1, 1, 640, 4, 5, 0)),
    ("one item", (1, 1, 1, 1, 64), (1, 1, 1, 1, 1, 1, 2)),
    ("131 items", (1, 1, 192 * 130 + 1, 200, 64), (131, 1, 1, 131, 1, 1, 2)),
    ("133 items", (1, 1, 192 * 132 + 129, 200, 64), (132, 1, 1, 133, 1, 2, 0)),
    ("1059 items", (1, 1, 192 * 1058 + 128, 200, 64), (132, 1, 1, 1059, 8, 9, 1)),
    ("VAE mid-block, 512x384", (8, 1, 3072, 3072, 512), (24, 4, 8, 768, 1, 1, 0)),
    ("VAE mid-block at d = 256, 64 queries", (3, 1, 64, 150, 256), (1, 2, 3, 6, 1, 1, 1)),
]


@pytest.mark.parametrize("name,shape,want", PLAN_TABLE, ids=[t[0] for t in PLAN_TABLE])
def test_plan_table(name, shape, want):
    B, heads, nq, nkv, D = shape
    p, err = plan_of(attn_desc(*shape), D != 64, SMS)
    assert p is not None, err
    got = tuple(p[k] for k in ("grid_x", "grid_y", "grid_z", "n_items", "items_min", "items_max", "idle_consumers_last_q_tile"))
    assert got == want and p == expected_plan(B, heads, nq, nkv, D, SMS), p


def test_census_plan_table():
    """Every attention descriptor of the workload census, with its pitches and batch strides on fake addresses, at 132 SMs."""
    desc, _, _ = census()
    rows = []
    for key, e in desc.items():
        if e["kind"] not in ("attn_d64", "attn_d512"):
            continue
        f = e["f"]
        D = f["d"]
        d = attn_desc(f["batch"], f["heads"], f["nq"], f["nkv"], D=D, q_pitch=f["qp"], q_batch_stride=f["qbs"], k_pitch=f["kp"],
                      k_batch_stride=f["kbs"], v_pitch=f["vp"], v_batch_stride=f["vbs"], out_pitch=f["op"], out_batch_stride=f["obs"])
        p = check_plan(d, dict(B=f["batch"], heads=f["heads"], nq=f["nq"], nkv=f["nkv"], D=D, want={}), SMS)
        rows.append(f"  D={D:3d} B={f['batch']:2d} heads={f['heads']:2d} nq={f['nq']:5d} nkv={f['nkv']:5d}: grid {p['grid_x']}x{p['grid_y']}x"
                    f"{p['grid_z']}, {p['n_items']} items ({p['items_min']}-{p['items_max']} per CTA), {p['n_kv_tiles']} key tiles   "
                    f"[{e['first']}]")
    print("\nattention plans of the workload census at 132 SMs\n" + "\n".join(rows))
    assert len(rows) >= 10 and any("D=512" in r for r in rows)


@pytest.mark.parametrize("case_id,case", all_cases(SMS), ids=[c[0] for c in all_cases(SMS)])
def test_case_plan_table(case_id, case):
    """The plan each GPU case targets, at 132 SMs (on a 132-SM H100 SXM also the plan that runs)."""
    p = check_plan(attn_desc(case["B"], case["heads"], case["nq"], case["nkv"], D=case.get("D", 64)), case, SMS)
    if case_id.startswith("items"):
        assert p["items_max"] == cdiv(p["n_items"], SMS)
    if case_id == "items 8sms+3":
        assert (p["items_min"], p["items_max"]) == (8, 9)  # items 0 .. 8 of a CTA: the Q buffer phase wraps twice


def test_ring_and_turn_residues_covered():
    """Over the ring cases' first five items per CTA, items start at every ring stage and phase (tile counter mod 8) and with every
    consumer warpgroup holding the turn (an item takes n_kv_tiles + 1 turns)."""
    stage, turn = set(), set()
    for n in N_TILES:
        assert expected_plan(**{k: ring_case(n, SMS)[k] for k in ("B", "heads", "nq", "nkv")}, D=64, n_sms=SMS)["items_min"] >= 5
        for i in range(5):
            stage.add(i * n % 8)
            turn.add(i * (n + 1) % 3)
    assert stage == set(range(8)) and turn == set(range(3))


def test_ops_attention_plan():
    """ops.attention_plan on the UNet's fused-QKV views (host tensors: the query reads no memory)."""
    from ladi_vton_b200 import ops
    qkv = torch.empty((16, 3072, 3 * 320), dtype=torch.bfloat16)
    p = ops.attention_plan(qkv[..., :320], qkv[..., 320:640], qkv[..., 640:], 5, SCALE, sms=132)
    assert (p.grid_x, p.n_items, p.items_min, p.items_max, p.n_kv_tiles) == (132, 1280, 9, 10, 24)
    x = torch.empty((2, 3072, 512), dtype=torch.bfloat16)
    p = ops.attention_plan(x, x, x, 1, 512 ** -0.5, wide=True, sms=132)
    assert (p.head_dim, p.grid_x, p.grid_y, p.grid_z) == (512, 24, 4, 2)
    with pytest.raises(RuntimeError, match="k_batch_stride"):
        k = torch.empty((16 * (77 * 320 + 4),), dtype=torch.bfloat16).as_strided((16, 77, 320), (77 * 320 + 4, 320, 1))
        ops.attention_plan(qkv[..., :320], k, k, 5, SCALE, sms=132)


# ================================================================================================================ CPU: the bound has teeth
TEETH_NKV = {"randn": 300, "late": 6, "early": 300, "tail": 300, "flat": 20, "level": 300}  # late: key tiles
# the faults each distribution is built to expose (emulate_attn's docstring)
EXPOSES = {"late": ["late", "l", "o", "quad"], "early": ["quad"], "tail": ["mask", "padded"], "flat": ["mask", "padded"]}


def _teeth_case(dist, tile, seed=4):
    nkv = TEETH_NKV[dist] * (tile if dist == "late" else 1)
    q, k, v = attn_inputs(dist, torch.Generator().manual_seed(seed), 1, 2, 96, nkv, 64, SCALE, tile)
    return q[0], k[0], v[0], nkv


def _teeth_worst(dist, tile, fault):
    q, k, v, nkv = _teeth_case(dist, tile)
    worst = 0.0
    for h in range(2):
        cs = slice(64 * h, 64 * h + 64)
        o, sv = attn_ref(q[:, cs].double(), k[:, cs].double(), v[:, cs].double(), 1, 64, SCALE)
        worst = max(worst, float(ratio(emulate_attn(q[:, cs], k[:, cs], v[:, cs], SCALE, tile, fault), o, attn_expect(o, sv, nkv)).max()))
    return worst


@pytest.mark.parametrize("tile", [128, 64])
@pytest.mark.parametrize("dist", ATTN_DISTS)
def test_bound_accepts_honest_attention(dist, tile):
    assert _teeth_worst(dist, tile, None) <= 1.0


FAULT_CASES = [(dist, fault) for dist, faults in EXPOSES.items() for fault in faults]


@pytest.mark.parametrize("tile", [128, 64])
@pytest.mark.parametrize("dist,fault", FAULT_CASES, ids=[f"{d}-{f}" for d, f in FAULT_CASES])
def test_bound_rejects_attention_faults(dist, fault, tile):
    """late: a skipped or late rescale of l or O, and a per-lane maximum; early: a per-lane maximum; tail / flat: the ragged mask off by
    one key and every padded key counted."""
    assert _teeth_worst(dist, tile, fault) > 1.0


@pytest.mark.parametrize("tile", [128, 64])
def test_score_distributions_do_what_they_say(tile):
    """late: every row's maximum rises on every key tile; early: tile 0 holds every row's maximum, >= 40 above every other key; tail:
    the last key holds every row's maximum; flat: all scores 0; level: one offset per (image, head), spread over [-48, 48]."""
    c = SCALE * 1.4426950408889634
    for dist in ("late", "early", "tail", "flat"):
        q, k, _, nkv = _teeth_case(dist, tile)
        x = (q[:, :64].double() @ k[:, :64].double().t()) * c
        if dist == "late":
            mx = torch.stack([x[:, j:j + tile].amax(1) for j in range(0, nkv, tile)], 1)
            assert bool((mx[:, 1:] > mx[:, :-1]).all())
        elif dist == "early":
            top = x.amax(1)
            assert bool((x[:, :tile].amax(1) == top).all()) and float((top - x.topk(2, dim=1).values[:, 1]).min()) >= 40
        elif dist == "tail":
            assert bool((x.argmax(1) == nkv - 1).all())
        else:
            assert float(x.abs().max()) == 0.0
    q, k, _ = attn_inputs("level", torch.Generator().manual_seed(4), 2, 3, 50, 100, 64, SCALE, tile)
    means = sorted(float((q[b, :, 64 * h:64 * h + 64].double() @ k[b, :, 64 * h:64 * h + 64].double().t()).mean()) * c
                   for b in range(2) for h in range(3))
    assert means[0] < -40 and means[-1] > 40


# ================================================================================================================ GPU: head width 64
@pytest.mark.gpu
@pytest.mark.parametrize("n_tiles", [1, 2, 3, 4, 24])
def test_key_tile_counts(cuda, n_tiles):
    run_case(Replay(cuda, 10 + n_tiles), 2, 2, 200, 128 * n_tiles)


@pytest.mark.gpu
@pytest.mark.parametrize("nkv", [77, 129, 255])
def test_ragged_last_key_tile(cuda, nkv):
    run_case(Replay(cuda, 40 + nkv), 2, 3, 192, nkv)


@pytest.mark.gpu
@pytest.mark.parametrize("nq", [1, 48, 64, 65, 128, 200, 260, 383])
def test_query_tails(cuda, nq):
    run_case(Replay(cuda, 70 + nq), 3, 2, nq, 300)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [96, 333])
def test_fused_qkv_in_place(cuda, n):
    run_case(Replay(cuda, 90 + n), 2, 5, n, n, fused=True)


@pytest.mark.gpu
@pytest.mark.parametrize("B, heads, nq, nkv", [(8, 8, 400, 300), (16, 10, 200, 77), (6, 5, 1000, 129)])
def test_persistent_ctas_run_several_items(cuda, B, heads, nq, nkv):
    # more (query tile, head, image) items than an H100 has SMs: CTAs carry the K / V ring, the Q double buffer and the warpgroups'
    # issue order from one item into the next
    run_case(Replay(cuda, B * heads + nq + nkv), B, heads, nq, nkv)


def _run(cuda, seed, case):
    run_case(Replay(cuda, seed), case["B"], case["heads"], case["nq"], case["nkv"], fused=case.get("fused", False), D=case.get("D", 64),
             dist=case.get("dist", "randn"), want=case["want"])


@pytest.mark.gpu
@pytest.mark.parametrize("label", list(ITEMS))
def test_items_against_sms(cuda, label):
    """1, sms - 1, sms, sms + 1, 2 sms + 1, 4 sms + 1 and 8 sms + 3 work items, hit exactly through the number of query tiles."""
    _run(cuda, 700 + list(ITEMS).index(label), items_case(label, sms(cuda)))


@pytest.mark.gpu
@pytest.mark.parametrize("n_tiles", N_TILES)
def test_ring_and_turn_residues(cuda, n_tiles):
    """n_tiles key tiles per item at >= 5 items per CTA: the ring stage and phase and the turn carry across items."""
    case = ring_case(n_tiles, sms(cuda))
    _run(cuda, 720 + n_tiles, dict(case, want=dict(case["want"], items_min=None)))
    assert expected_plan(case["B"], case["heads"], case["nq"], case["nkv"], 64, sms(cuda))["items_min"] >= 5


@pytest.mark.gpu
@pytest.mark.parametrize("r", list(TAIL_IDLE))
def test_query_tails_multi_item(cuda, r):
    """nq mod 192 = r at >= 3 items per CTA: CTAs alternate full items with items whose last consumers have no or few rows."""
    case = tail_case(r, sms(cuda))
    _run(cuda, 740 + r, dict(case, want=dict(case["want"], items_min=None)))
    assert expected_plan(case["B"], case["heads"], case["nq"], case["nkv"], 64, sms(cuda))["items_min"] >= 3


@pytest.mark.gpu
@pytest.mark.parametrize("placement", PLACEMENTS)
@pytest.mark.parametrize("dist", ATTN_DISTS)
def test_score_distributions(cuda, dist, placement):
    case = dist_case(dist, placement, sms(cuda))
    _run(cuda, 800 + 10 * ATTN_DISTS.index(dist) + PLACEMENTS.index(placement), dict(case, dist=dist, want={
        k: v for k, v in case["want"].items() if v is not None}))


@pytest.mark.gpu
def test_late_maximum_96_key_tiles(cuda):
    """The maximum moves up on each of 96 key tiles (12288 keys, the 1024x768 level-0 length)."""
    run_case(Replay(cuda, 900), 1, 2, 400, 12288, dist="late", want=dict(n_kv_tiles=96))


# ================================================================================================================ head width 512 / 256
# attention_kernel<D>: 128-row query tiles over two consumer warpgroups (64 rows each), 64-key tiles, a 10-stage ring of 64-column
# chunks that one D = 512 tile fills exactly (8 K + 2 V chunks) and a D = 256 tile (4 + 2) wraps mid-tile, TMA zero-fill at nq / nkv.
@pytest.mark.gpu
@pytest.mark.parametrize("D", [512, 256])
@pytest.mark.parametrize("nkv", [1, 63, 64, 65, 127, 64 * 101 + 5])
def test_wide_key_counts(cuda, D, nkv):
    run_case(Replay(cuda, 200 + nkv + D), 3, 1, 130, nkv, D=D)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [512, 256])
@pytest.mark.parametrize("nq", [1, 63, 64, 65, 127, 128, 129])
def test_wide_query_tails(cuda, D, nq):
    # nq = 1 .. 64: the second consumer warpgroup of the only query tile has no rows; 65: one
    run_case(Replay(cuda, 300 + nq + D), 3, 1, nq, 150, D=D, want=dict(idle_consumers_last_q_tile=1 if nq % 128 in range(1, 65) else 0))


@pytest.mark.gpu
@pytest.mark.parametrize("D", [512, 256])
def test_wide_fused_qkv_in_place(cuda, D):
    run_case(Replay(cuda, 400 + D), 3, 1, 200, 200, fused=True, D=D)


@pytest.mark.gpu
@pytest.mark.parametrize("n_tiles", [1, 2, 5, 40])
def test_d256_ring_wraps(cuda, n_tiles):
    # 6 ring stages per key tile of 10: the ring wraps mid-tile from the second tile on
    run_case(Replay(cuda, 500 + n_tiles), 3, 1, 160, 64 * n_tiles, D=256)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [512, 256])
def test_wide_late_maximum(cuda, D):
    run_case(Replay(cuda, 600 + D), 3, 1, 200, WIDE_DIST_NKV["late"], D=D, dist="late")


@pytest.mark.gpu
@pytest.mark.parametrize("D", [512, 256])
@pytest.mark.parametrize("dist", ["early", "tail", "flat", "level"])
def test_wide_score_distributions(cuda, dist, D):
    run_case(Replay(cuda, 620 + D + ATTN_DISTS.index(dist)), 3, 1, 200, WIDE_DIST_NKV[dist], D=D, dist=dist)
