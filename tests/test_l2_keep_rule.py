"""Host-side restatement of the L2 residency rule of the attention launches (latex_ocr_b200/csrc/lo_attention.cu: att_keep_stage,
att_keep_q): which ring stages of a CTA are kept in L2 for a budget of att_l2_keep_mb MiB.  Checked over the launch geometries the
decoder uses (cfg #2, cfg #4, ragged and beam decode): the kept bytes never exceed the budget, budget 0 keeps nothing, a huge budget
keeps every stage after the ring depth, and the kept stages are spread evenly.  Pure Python: runs without a GPU."""
import pytest

L2_BYTES = 50 << 20        # H100 SXM
NUM_SMS, MINB, MAXSPLIT = 132, 2, 16


def keep_stage(i, depth, q):
    j = i - depth
    return j >= 0 and ((j + 1) * q) >> 10 != (j * q) >> 10


def keep_q(budget_mb, nbytes, l2=L2_BYTES):
    budget = min(budget_mb << 20, l2)
    if budget <= 0 or nbytes <= 0:
        return 0
    return min(1024, budget * 1024 // nbytes)


def splits(B):
    return max(1, min(MAXSPLIT, NUM_SMS * MINB // B))


def fwd_ctas(R, ns, rows=16):
    """(rows streamed, stages) of every split of one batch row in the forward pipe kernel"""
    rps = (R + ns - 1) // ns
    out = []
    for sp in range(ns):
        r0, r1 = sp * rps, min(R, sp * rps + rps)
        n = r1 - r0 if r1 > r0 else 0
        out.append((n, (n + rows - 1) // rows))
    return out


def bwd_ctas(R, ns, rows=16):
    rps = (((R + ns - 1) // ns) + 1) & ~1
    out = []
    for sp in range(ns):
        r0, r1 = sp * rps, min(R, sp * rps + rps)
        n = r1 - r0 if r1 > r0 else 0
        out.append((n, (n + rows - 1) // rows))
    return out


def kept_rows(n_rows, nst, depth, q, rows=16):
    return sum(min(rows, n_rows - i * rows) for i in range(nst) if keep_stage(i, depth, q))


# (launch, images, rows per image, regions per image, bytes per region row, stage depth)
LAUNCHES = [
    ("cfg2 forward", 64, 1, [868] * 64, 2048, 3),
    ("cfg2 backward", 64, 1, [868] * 64, 1024, 5),
    ("cfg4 forward", 20, 1, [1404] * 20, 2048, 3),
    ("cfg4 backward", 20, 1, [1404] * 20, 1024, 5),
    ("beam decode forward", 8, 5, [868] * 8, 2048, 3),
    ("ragged decode forward", 6, 1, [40, 868, 101, 1404, 16, 300], 2048, 3),
]


def _launch_kept_bytes(n_img, rpi, regions, row_bytes, depth, budget_mb):
    B = n_img * rpi
    ns = splits(B)
    q = keep_q(budget_mb, sum(regions) * row_bytes)          # distinct rows: the rows of an image are read by its rpi rows alike
    kept = 0
    for R in regions:                                          # one image: its rows share the split geometry and so the kept set
        geo = fwd_ctas(R, ns) if depth == 3 else bwd_ctas(R, ns)
        kept += sum(kept_rows(n, nst, depth, q) for n, nst in geo) * row_bytes
    return kept, q


@pytest.mark.parametrize("name,n_img,rpi,regions,row_bytes,depth", LAUNCHES, ids=[x[0] for x in LAUNCHES])
@pytest.mark.parametrize("budget_mb", [0, 1, 8, 13, 16, 24, 32, 40, 50, 4096])
def test_kept_bytes_never_exceed_the_budget(name, n_img, rpi, regions, row_bytes, depth, budget_mb):
    kept, q = _launch_kept_bytes(n_img, rpi, regions, row_bytes, depth, budget_mb)
    assert kept <= min(budget_mb << 20, L2_BYTES)
    if budget_mb == 0:
        assert q == 0 and kept == 0


def test_a_budget_that_covers_the_launch_keeps_every_stage_after_the_ring_depth():
    for nst in range(0, 40):
        for depth in (3, 5):
            assert [keep_stage(i, depth, 1024) for i in range(nst)] == [i >= depth for i in range(nst)]
    # 40 images of 101 regions: 8.3 MB, under the default budget
    assert keep_q(24, 40 * 101 * 2048) == 1024


def test_budget_is_clamped_to_the_l2():
    assert keep_q(4096, 10 << 30) == keep_q(50, 10 << 30)
    assert keep_q(-3, 1 << 20) == 0


@pytest.mark.parametrize("q", [1, 100, 226, 333, 512, 700, 1023])
def test_kept_stages_are_spread_evenly(q):
    depth, n = 3, 200
    kept = [i - depth for i in range(depth + n) if keep_stage(i, depth, q)]
    assert len(kept) == n * q // 1024
    # every window of w consecutive eligible stages holds floor or ceil of w * q / 1024 kept stages
    for w in (4, 11, 37):
        for s in range(0, n - w + 1):
            c = sum(1 for j in kept if s <= j < s + w)
            assert w * q // 1024 <= c <= -(-w * q // 1024)
