"""CPU model of the MMA warpgroup's fragment walk (banet_b200/csrc/mma_role.cuh) on the 128-B swizzled tiles (tc_utils.cuh: frag_off).

Proves on the host what the kernel relies on: its lane offsets address exactly the columns of the fragment <-> column mapping, the
accumulators of each warp cover the lower block triangle of H_dd plus the [v | t] columns exactly once, the span write inverts the
mapping, and the LDS.128 walk of R is bank-conflict-free per quarter-warp (the LDS.64 walks of A keep the 2-way conflict that no
walk over one 16-column m-block avoids)."""
import itertools

import pytest


def frag_off(col, r):                          # tc_utils.cuh: byte offset of (pixel row r of a step, column col)
    return (col >> 5) * 8192 + r * 128 + ((((col & 31) >> 2) ^ r) << 4) + (col & 3) * 4


def lane_offsets(lane, KR):                    # mma_role.cuh: mma_warp
    g, t = lane >> 2, lane & 3
    oa = t * 128 + (((g >> 1) ^ t) << 4) + (g & 1) * 8
    ob0 = t * 128 + ((((g >> 1) | ((g & 1) << 2)) ^ t) << 4)
    ob1 = (ob0 ^ 64) + 512
    ox = (KR // 32) * 8192 + t * 128 + (((g >> 2) ^ t) << 4) + (g & 3) * 4
    return oa, ob0, ob1, ox


def full_groups(mb):
    return 0 if mb < 0 else (mb + 1) // 2


def half_group(mb):
    return mb >= 0 and mb % 2 == 0


def split(KR):                                 # mma_role.cuh: mma_role
    if KR == 128:
        return [(0, 7), (1, 6), (2, 5), (3, 4)]
    return [(mw if mw < KR // 16 else -1, -1) for mw in range(4)]


def c(g):
    return (g >> 1) | ((g & 1) << 2)


def loads(mb, lane, KR):
    """Every load of one 8-pixel step for m-block mb: (kind, byte offset as the kernel forms it, [(pixel row, column) per 4-B word])."""
    g, t = lane >> 2, lane & 3
    oa, ob0, ob1, ox = lane_offsets(lane, KR)
    out = []
    out.append(("A", (mb >> 1) * 8192 + oa + 64 * (mb & 1), [(t, 16 * mb + 2 * g), (t, 16 * mb + 2 * g + 1)]))
    out.append(("A", (mb >> 1) * 8192 + 512 + oa + 64 * ((mb & 1) ^ 1), [(t + 4, 16 * mb + 2 * g), (t + 4, 16 * mb + 2 * g + 1)]))
    for G in range(full_groups(mb)):
        out.append(("R", G * 8192 + ob0, [(t, 32 * G + 4 * c(g) + j) for j in range(4)]))
        out.append(("R", G * 8192 + ob1, [(t + 4, 32 * G + 4 * c(g) + j) for j in range(4)]))
    if half_group(mb):
        G = full_groups(mb)
        out.append(("R", G * 8192 + oa, [(t, 32 * G + 2 * g + j) for j in range(2)]))
        out.append(("R", G * 8192 + 512 + oa + 64, [(t + 4, 32 * G + 2 * g + j) for j in range(2)]))
    out.append(("X", ox, [(t, KR + g)]))
    out.append(("X", ox + 576, [(t + 4, KR + g)]))
    return out


def accumulators(mb, lane, KR):
    """(row i, column n) of every accumulator element of m-block mb in this lane, as the span write places it."""
    g, t = lane >> 2, lane & 3
    out = []
    for e in range(4):
        i = 16 * mb + 2 * g + (e >> 1)
        out += [(i, 32 * G + 16 * (e & 1) + 4 * t + j) for G in range(full_groups(mb)) for j in range(4)]
        if half_group(mb):
            out += [(i, 32 * full_groups(mb) + 2 * (e & 1) + 4 * t + j) for j in range(2)]
        out.append((i, KR + 2 * t + (e & 1)))
    return out


def mma_element(row_of, col_of):
    """m16n8k8 fragment roles (PTX ISA): lane (g, t) holds A rows g / g+8 at k = t / t+4, B column g at k = t / t+4, and the
    accumulator element e at row g + 8(e >> 1), column 2t + (e & 1).  Given the basis column of each fragment row and the R column of
    each fragment column, return {(lane, e): (basis column, R column)} of the accumulator."""
    return {(lane, e): (row_of((lane >> 2) + 8 * (e >> 1)), col_of(2 * (lane & 3) + (e & 1)))
            for lane in range(32) for e in range(4)}


@pytest.mark.parametrize("KR", [128, 64, 32])
def test_lane_offsets_address_the_mapped_columns(KR):
    for pair in split(KR):
        for mb in pair:
            if mb < 0:
                continue
            for lane in range(32):
                for kind, off, words in loads(mb, lane, KR):
                    for w, (r, col) in enumerate(words):
                        assert off + 4 * w == frag_off(col, r), (kind, mb, lane, w)


@pytest.mark.parametrize("KR", [128, 64, 32])
def test_fragment_roles_match_the_accumulator_mapping(KR):
    """The element the tensor core forms at (lane, e) is (basis column, R column) = what the span write says it is."""
    for pair in split(KR):
        for mb in pair:
            if mb < 0:
                continue
            row_of = lambda fr: 16 * mb + 2 * (fr & 7) + (fr >> 3)          # fragment row -> basis column
            blocks = [(lambda G, j: (lambda fc: 32 * G + 4 * c(fc) + j))(G, j) for G in range(full_groups(mb)) for j in range(4)]
            if half_group(mb):
                blocks += [(lambda G, j: (lambda fc: 32 * G + 2 * fc + j))(full_groups(mb), j) for j in range(2)]
            blocks.append(lambda fc: KR + fc)
            for lane in range(32):
                acc = accumulators(mb, lane, KR)
                formed = []
                for e in range(4):
                    for col_of in blocks:
                        el = mma_element(row_of, col_of)
                        formed.append(el[(lane, e)])
                assert sorted(formed) == sorted(acc)
                # the B words a lane loads are exactly the columns of its fragment column g in every block (b0 at t, b1 at t+4)
                g, t = lane >> 2, lane & 3
                got = sorted(col for kind, _, words in loads(mb, lane, KR) if kind != "A" for r, col in words if r == t)
                assert got == sorted(col_of(g) for col_of in blocks)


@pytest.mark.parametrize("KR", [128, 64, 32])
def test_accumulators_cover_the_block_triangle_once(KR):
    for pair in split(KR):
        written = []
        for mb in pair:
            if mb < 0:
                continue
            need = {(i, n) for i in range(16 * mb, 16 * mb + 16) for n in list(range(16 * mb + 16)) + list(range(KR, KR + 8))}
            got = [x for lane in range(32) for x in accumulators(mb, lane, KR)]
            assert len(got) == len(set(got)) and set(got) == need
            written += [(i, n) for i, n in got if n < KR or n - KR < 7]
        assert len(written) == len(set(written))
    allw = {x for pair in split(KR) for mb in pair if mb >= 0 for lane in range(32) for x in accumulators(mb, lane, KR)}
    assert {(i, n) for i, n in allw if n < KR} == {(i, n) for i in range(KR) for n in range(KR) if n // 16 <= i // 16}


def _banks(off, nbytes):
    return {((off + b) % 128) // 4 for b in range(0, nbytes, 4)}


def test_r_group_loads_are_conflict_free_and_a_loads_two_way():
    """LDS.128 is served per quarter-warp (8 lanes x 16 B), LDS.64 per half-warp (16 lanes x 8 B): count the wavefronts."""
    for mb, kk in itertools.product(range(8), range(8)):
        per_lane = [loads(mb, lane, 128) for lane in range(32)]
        for k, (kind, _, words) in enumerate(per_lane[0]):
            width = 4 * len(words)
            phase = 128 // width
            for p0 in range(0, 32, phase):
                lanes = range(p0, p0 + phase)
                use = {}
                for ln in lanes:
                    off = kk * 1024 + per_lane[ln][k][1]
                    for b in _banks(off, width):
                        use.setdefault(b, set()).add(off // 128)
                ways = max(len(v) for v in use.values())
                if kind == "R" and width == 16:
                    assert ways == 1, (mb, kk, k)
                elif kind == "A" or (kind == "R" and width == 8):
                    assert ways == 2, (mb, kk, k)
