"""CPU side of test_gemm_epilogue_bits_gpu.py: the row-statistics statement has teeth, reproduces a hand-worked example, and the
sweep's case list covers every axis it claims to.

The summation-tree mutants below are the plausible ways an epilogue rewrite could reorder the sums while every tolerance-based test
keeps passing: chunks walked in ascending order (so a half no longer holds the chunks of one parity), a plain left-to-right column
sum, the xor fold pairing groups (0, 2) and (1, 3), and the two 16-column halves of a chunk added the other way round.
"""
import torch

from tests.test_gemm_epilogue_bits_gpu import (EPILOGUES, FLAT_EPIS, GLU_EPIS, GLU_TILES, M_LIST, RESIDUES, SPECIALISED_O16, SWEEP_GROUPS,
                                               WIDE_EPIS, WIDTHS, specialised_cases, stats_statement, sweep_cases)
from tests.test_gemm_schedule_gpu import fma32
from tests.test_kernel_variants_gpu import MODES, VARIANTS

H100_SMS = 132


def tree(x, BN, bn_out, order="documented"):
    """[M, tiles * bn_out] fp32 rows (whole tiles) -> [M, 2 * tiles, 2] partials, summed in `order`: 'documented', 'ascending'
    (chunk_of(k) = k: the first (NCH + 1) / 2 chunks of the BN-wide tile fill half 0), 'left-to-right' (each half's columns one
    by one, s1 += x, s2 = fma(x, x, s2)), 'fold-02-13' ((S0 + S2) + (S1 + S3)) or 'halves-swapped' ((S + q(k, kc + 4)) + q(k, kc))."""
    M, n = x.shape
    tiles, nlive, nch = n // bn_out, bn_out // 32, BN // 32
    nev = (nch + 1) // 2
    if order == "ascending":
        halves = [[k for k in range(nev) if k < nlive], [k for k in range(nev, nch) if k < nlive]]
    else:
        halves = [list(range(0, nlive, 2)), list(range(1, nlive, 2))]
    xc = x.view(M, tiles, nlive, 32)
    out = torch.zeros(M, tiles, 2, 2, dtype=torch.float32)
    for h, chunks in enumerate(halves):
        if order == "left-to-right":
            s1 = s2 = torch.zeros(M, tiles, dtype=torch.float32)
            for k in chunks:
                for c in range(32):
                    v = xc[:, :, k, c]
                    s1, s2 = s1 + v, fma32(v, v, s2)
            out[:, :, h, 0], out[:, :, h, 1] = s1, s2
            continue
        o0, o1, o2, o3 = xc.view(M, tiles, nlive, 8, 4).unbind(-1)
        qs = ((o0 + o1) + (o2 + o3), fma32(o0, o0, o1 * o1) + fma32(o2, o2, o3 * o3))
        for j, q in enumerate(qs):
            s = torch.zeros(M, tiles, 4, dtype=torch.float32)
            for k in chunks:
                a, b = (q[:, :, k, 4:], q[:, :, k, :4]) if order == "halves-swapped" else (q[:, :, k, :4], q[:, :, k, 4:])
                s = (s + a) + b
            if order == "fold-02-13":
                out[:, :, h, j] = (s[..., 0] + s[..., 2]) + (s[..., 1] + s[..., 3])
            else:
                out[:, :, h, j] = (s[..., 0] + s[..., 1]) + (s[..., 2] + s[..., 3])
    return out.view(M, 2 * tiles, 2)


def bits(t):
    return t.contiguous().view(torch.int32)


def test_statement_has_teeth():
    """On random rows of 128-wide tiles, each wrong order changes the bits of a large share of the (row, part) entries, and an
    independent loop over the documented order agrees with stats_statement bit for bit."""
    g = torch.Generator().manual_seed(11)
    M, tiles, bn = 256, 3, 128
    x = (torch.randn(M, tiles * bn, generator=g) * 2.0 + 0.7).float()
    want = stats_statement(x, M, tiles * bn, bn, 2 * tiles)
    assert torch.equal(bits(tree(x, bn, bn)), bits(want))
    shares = {}
    for order in ("ascending", "left-to-right", "fold-02-13", "halves-swapped"):
        diff = (bits(tree(x, bn, bn, order)) != bits(want)).any(-1)
        shares[order] = diff.double().mean().item()
    print(f"\nshare of (row, part) entries whose bits differ from the documented tree: {shares}")
    for order, share in shares.items():
        assert share > 0.3, (order, shares)
    # the 96-wide tile (three chunks: half 0 = chunks 0 and 2) separates the chunk orders too; the 64-wide one cannot
    x96 = x[:, :192].contiguous()
    want96 = stats_statement(x96, M, 192, 96, 4)
    assert (bits(tree(x96, 96, 96, "ascending")) != bits(want96)).any(-1).double().mean().item() > 0.3
    assert (bits(tree(x96, 96, 96, "halves-swapped")) != bits(want96)).any(-1).double().mean().item() > 0.1
    x64 = x[:, :128].contiguous()
    for order in ("ascending", "halves-swapped"):  # one chunk per half: these orders coincide with the documented one
        assert torch.equal(bits(tree(x64, 64, 64, order)), bits(stats_statement(x64, M, 128, 64, 4)))


def test_statement_hand_worked_example():
    """One row, two 64-wide n-tiles, n_out = 92: the second tile's last 4-column group is past n_out and its odd chunk is
    empty.  Worked by hand:
      part 0 (tile 0, chunk 0): columns 0, 4, 8, 12 = 2^25, 2, 1, 1 are groups kc = 0..3 of the first 16-column half, so
        S = (2^25, 2, 1, 1) and the sum is (2^25 + 2) + (1 + 1) = 2^25 + 2 = 2^25 (a tie, to the even neighbour; fp32 spacing
        at 2^25 is 4).  The sum of squares: (2^50 + 4) + 2 = 2^50.  (The fold (S0 + S2) + (S1 + S3) gives 2^25 + 3 = 2^25 + 4.)
      part 1 (tile 0, chunk 1): columns 32, 33, 63 = 0.5, -0.25, 0.75: groups 0 and 7, sum 0.25 + 0.75 = 1, sum of squares
        fma(0.5, 0.5, 0.0625) + fma(0, 0, 0.5625) = 0.875.
      part 2 (tile 1, chunk 0, columns 64 .. 91 live): columns 88, 91 = 3, 1 (group 6): sum 4, sum of squares 10.
      part 3 (tile 1, chunk 1, no live column): (+0, +0)."""
    x = torch.zeros(1, 92)
    for c, v in ((0, 2.0 ** 25), (4, 2.0), (8, 1.0), (12, 1.0), (32, 0.5), (33, -0.25), (63, 0.75), (88, 3.0), (91, 1.0)):
        x[0, c] = v
    got = stats_statement(x, 1, 92, 64, 4)
    want = torch.tensor([[[2.0 ** 25, 2.0 ** 50], [1.0, 0.875], [4.0, 10.0], [0.0, 0.0]]])
    assert torch.equal(bits(got), bits(want)), got
    padded = torch.cat([x, torch.zeros(1, 36)], 1)
    assert tree(padded, 64, 64, "fold-02-13")[0, 0, 0].item() == 2.0 ** 25 + 4
    assert x.double().sum().item() == 2.0 ** 25 + 9.0  # the exact sum: the tree's rounding is part of the contract


def test_sweep_epilogues_are_what_they_claim():
    """The v.. epilogues are the VIMA_GEMM_VARIANTS rows of that index (test_variant_table_matches_the_compiled_list holds VARIANTS
    to the compiled list), the generic ones are none of its rows, and SPECIALISED_O16 is every row with a 16-bit output and no fp32
    one."""
    for name, row in EPILOGUES.items():
        if name.startswith("v"):
            assert VARIANTS[int(name[1:3])] == row, name
        else:
            assert name.startswith("generic-") and row not in VARIANTS, name
        assert row[4], f"{name}: every sweep call writes out_f32"
        assert row[5] or row[8], f"{name}: and at least one other output"
    assert set(WIDE_EPIS) <= {k for k in EPILOGUES if k.startswith("v")}
    assert SPECIALISED_O16 == [i for i, r in enumerate(VARIANTS) if r[5] and not r[4]]
    for i in SPECIALISED_O16:  # with out_f32 added the descriptor runs the generic epilogue
        assert VARIANTS[i][:4] + (1,) + VARIANTS[i][5:] not in VARIANTS


def dead_and_partial(c):
    """(parities of whole dead chunks, parities of partly live chunks) in the case's last n-tile."""
    r = c["n_out"] - (c["n_out"] - 1) // c["bn"] * c["bn"]
    dead = {k % 2 for k in range(c["bn"] // 32) if 32 * k >= r}
    partial = {k % 2 for k in range(c["bn"] // 32) if 32 * k < r < 32 * (k + 1)}
    return dead, partial


def test_sweep_covers_every_axis():
    """Every value of every axis at least once, in the combinations where it matters, in a bounded number of cases."""
    cases = [c for grp in SWEEP_GROUPS for c in sweep_cases(grp)]
    assert len(cases) < 400, len(cases)
    assert cases == [c for grp in SWEEP_GROUPS for c in sweep_cases(grp)], "deterministic"
    tc = [c for c in cases if not c["wide"]]
    wide = [c for c in cases if c["wide"]]
    for mode in MODES:
        for key in WIDTHS:
            sel = [c for c in tc if c["mode"] == mode and c["width"] == key]
            assert sel, (mode, key)
            if key.isdigit():
                assert sorted(c["residue"] for c in sel) == [r for r in RESIDUES if r <= int(key)], (mode, key)
            for epi in (GLU_EPIS if key.startswith("glu") else []):
                assert any(c["epi"] == epi for c in sel), (mode, key, epi)
        assert {c["epi"] for c in tc if c["mode"] == mode} == set(EPILOGUES), mode
    for key in WIDTHS:
        sel = [c for c in tc if c["width"] == key]
        assert {c["M"] for c in sel} == set(M_LIST), key
        bn = sel[0]["bn"]
        bn_out = bn // 2 if key.startswith("glu") else bn
        ntiles = {-(-c["n_out"] // bn_out) for c in sel}
        assert 1 in ntiles and max(ntiles) > 2, (key, ntiles)
        assert any(-(-c["M"] // 128) * -(-c["n_out"] // bn_out) > H100_SMS for c in sel), f"{key}: no CTA walks several tiles"
        if key.startswith("glu"):
            assert ntiles >= set(GLU_TILES), key
            continue
        assert {c["epi"] for c in sel} == set(FLAT_EPIS), key
        for epi in FLAT_EPIS:
            row = EPILOGUES[epi]
            if row[2] or row[3]:  # reads multiplier / residual rows: the L2 prefetch both ways
                assert {c["prefetch"] for c in sel if c["epi"] == epi} == {0, 1}, (key, epi)
        dead = set().union(*(dead_and_partial(c)[0] for c in sel))
        partial = set().union(*(dead_and_partial(c)[1] for c in sel))
        assert dead == ({0, 1} if bn >= 96 else {1} if bn == 64 else set()), (key, dead)
        assert partial == ({0, 1} if bn >= 64 else {0}), (key, partial)
    # the wide kernel: only whole 256-wide tiles, its specialised epilogues, several tiles per CTA, both prefetch settings
    assert wide and all(c["mode"] == "f16f8" and c["bn"] == 128 and c["n_out"] % 256 == 0 for c in wide)
    assert {c["epi"] for c in wide} == set(WIDE_EPIS) and {c["prefetch"] for c in wide} == {0, 1}
    assert any(-(-c["M"] // 128) * (c["n_out"] // 256) > H100_SMS for c in wide)
    # section 3: every O16-only row on every tile width it takes, at a multi-tile M
    for i in SPECIALISED_O16:
        sc = specialised_cases(i)
        assert {bn for _, _, bn, _ in sc} == ({64, 128} if VARIANTS[i][1] else {32, 64, 96, 128}), i
        assert any(M > 128 * 8 for M, _, _, _ in sc), i
