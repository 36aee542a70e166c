"""The head-width-64 attention kernel at the edges of its schedule: the QK^T pipeline's prologue and drain (1, 2, 3, 4 and 24 key tiles),
ragged last key tiles, query tails that leave some consumer warpgroups of the last query tile with few or no rows, and the fused-QKV
projection read in place.  Each case is checked the way the workload census checks the workload's calls (tests/kernel_check.py): against float64
with the same per-element bound, bit for bit against a second run, and with every byte of the output buffer outside the rows and columns
the call owns (pitch gaps, the gap between batch images) NaN-poisoned before the call and still NaN after it."""
import ctypes as C

import pytest
import torch

from kernel_check import Replay, attn_expect, attn_ref, max_ratio, same

SCALE = 0.125
PAD = 24  # columns of NaN after each row of every operand (keeps the pitch a multiple of 8)
GAP = 40  # NaN elements between consecutive batch images


def _operand(R, B, n, width, pitch, bstride, std, col0=0, buf=None):
    """values [B, n, width] written at column col0 of a [B] x [n rows of `pitch`] buffer with batch stride `bstride` (NaN elsewhere)."""
    if buf is None:
        buf = torch.full(((B - 1) * bstride + n * pitch,), float("nan"), dtype=torch.bfloat16, device=R.dev)
    vals = (R.randn(B, n, width) * std).bfloat16()
    buf.as_strided((B, n, width), (bstride, pitch, 1), col0).copy_(vals)
    return buf, vals


def _late_max_keys(R, B, nkv, D, scale):
    """Keys whose scores grow by 2 per 64-key tile along a direction every query shares: each tile holds a larger maximum than all
    before it, so the online softmax rescales l and O on every tile."""
    u = torch.sign(R.randn(D))
    k = (R.randn(B, nkv, D) * 0.5 + (2.0 * (torch.arange(nkv, device=R.dev) // 64) / (scale * D))[None, :, None] * u).bfloat16()
    return k, u


def run_case(R, B, heads, nq, nkv, fused=False, D=64, late_max=False):
    """D = 64: ladi_attention_bf16 with `heads` heads; D = 512 / 256: ladi_attention_d512_bf16 (heads must be 1, head_dim = D)."""
    from ladi_vton_b200 import lib
    width = heads * D
    scale = SCALE if D == 64 else D ** -0.5
    d = lib.AttnDesc()
    d.batch, d.heads, d.nq, d.nkv, d.scale, d.variant = B, heads, nq, nkv, scale, 0
    d.head_dim = 0 if D == 64 else D
    if fused:  # one [B][n][3 * width + PAD] projection output: q, k, v are column slices of it
        assert nq == nkv
        pitch = 3 * width + PAD
        bs = nq * pitch + GAP
        buf, q = _operand(R, B, nq, width, pitch, bs, 2 ** 0.5)
        _, k = _operand(R, B, nq, width, pitch, bs, 2 ** 0.5, col0=width, buf=buf)
        _, v = _operand(R, B, nq, width, pitch, bs, 1.0, col0=2 * width, buf=buf)
        base = buf.data_ptr()
        d.q, d.k, d.v = base, base + 2 * width, base + 4 * width
        d.q_pitch = d.k_pitch = d.v_pitch = pitch
        d.q_batch_stride = d.k_batch_stride = d.v_batch_stride = bs
        keep = [buf]
    else:
        pitch = width + PAD
        qb, q = _operand(R, B, nq, width, pitch, nq * pitch + GAP, 2 ** 0.5)
        kb, k = _operand(R, B, nkv, width, pitch, nkv * pitch + GAP, 2 ** 0.5)
        if late_max:
            k, u = _late_max_keys(R, B, nkv, D, scale)
            q = (q.float() * 0.5 + u).bfloat16()
            qb.as_strided((B, nq, width), (nq * pitch + GAP, pitch, 1)).copy_(q)
            kb.as_strided((B, nkv, width), (nkv * pitch + GAP, pitch, 1)).copy_(k)
        vb, v = _operand(R, B, nkv, width, pitch, nkv * pitch + GAP, 1.0)
        d.q, d.q_pitch, d.q_batch_stride = qb.data_ptr(), pitch, nq * pitch + GAP
        d.k, d.k_pitch, d.k_batch_stride = kb.data_ptr(), pitch, nkv * pitch + GAP
        d.v, d.v_pitch, d.v_batch_stride = vb.data_ptr(), pitch, nkv * pitch + GAP
        keep = [qb, kb, vb]
    op, obs = width + PAD, nq * (width + PAD) + GAP
    d.out_pitch, d.out_batch_stride = op, obs
    outs = []
    for _ in range(2):
        o = torch.full(((B - 1) * obs + nq * op,), float("nan"), dtype=torch.bfloat16, device=R.dev)
        d.out = o.data_ptr()
        lib.call("ladi_attention_bf16" if D == 64 else "ladi_attention_d512_bf16", C.byref(d), R.stream)
        outs.append(o)
    torch.cuda.synchronize()
    del keep
    out = outs[0]
    owned = torch.zeros(out.shape, dtype=torch.bool, device=R.dev)
    owned.as_strided((B, nq, width), (obs, op, 1)).fill_(True)
    assert bool(torch.isfinite(out[owned].float()).all()), "unwritten or NaN-contaminated output element"
    assert bool(torch.isnan(out[~owned].float()).all()), "wrote outside its rows and columns (pitch gap or batch gap)"
    assert same(outs[0], outs[1]), "two runs differ bitwise"
    ov = out.as_strided((B, nq, width), (obs, op, 1))
    for b in range(B):
        o64, sv = attn_ref(q[b].double(), k[b].double(), v[b].double(), heads, D, scale)
        worst = max_ratio(ov[b], o64, attn_expect(o64, sv, nkv))
        assert worst <= 1.0, f"image {b}: err/bound {worst:.3g}"


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
    run_case(Replay(cuda, 300 + nq + D), 3, 1, nq, 150, D=D)


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
    run_case(Replay(cuda, 600 + D), 3, 1, 200, 64 * 7 + 10, D=D, late_max=True)
