"""Python statement of how the build kernels split their tiles over a persistent grid and find the partial slots again.

Restates, without a GPU:
- `build_plan` (lm_build.cu), `build_plan_tc` (lm_build_tc_host.cu) and `keyframe_plan` (lm_window_key.cu): grid, tiles per pair
  (window), max_span, slot size and workspace bytes;
- `part_begin` (common.cuh): CTA c owns tiles [part_begin(c), part_begin(c + 1));
- the span walks of the build kernels: a CTA starts a new span (partial slot c * max_span + span) whenever the pair of its tile changes.
  lm_build_tc6_kernel counts spans in three roles on its own: the gather warps hand their |d| sums over at a pair change and at the end
  of the range (`dump_rb`), while the algebra and MMA warps flush at the last tile of a pair or of the range, tracked by a tile counter
  `rr` that starts at `(unsigned)t_begin % tiles_per_pair`;
- the reduce's slot search (`lm_reduce_kernel`, `keyframe_reduce_kernel`), one lane per pair.

tests/test_build_edges.py sweeps shapes through it and checks that every slot written is read exactly once, by its own pair."""
import numpy as np

TILE = 64                       # points per tile: TILE_PX (SIMT), TC_TILE (tensor cores), KT_PX (keyframe)
MAX_SMS = 132                   # kMaxSMs (common.cuh)
REDUCE_CAP = 2 * MAX_SMS + 8    # slots the reduce kernels can list for one pair


def _align_up(x, a):
    return (x + a - 1) // a * a


def slot_floats(K, C):
    return ((K * K + 7 * K + 32 + C) + 3) // 4 * 4                 # SlotLayout::floats


def key_slot_floats(K, C, nf):
    return K * K + nf * ((7 * K + 32 + C + 3) // 4 * 4)             # KeySlot::floats


def padded_K(K):
    for kp in (0, 16, 32, 64, 128, 256):
        if K <= kp:
            return kp
    return -1


class Plan:
    def __init__(self, total_tiles, tiles_per_pair, grid, slot, max_span_delta=0):
        grid = max(1, min(grid, total_tiles))
        tiles_per_cta = (total_tiles + grid - 1) // grid
        self.total_tiles, self.tiles_per_pair, self.grid, self.slot_floats = total_tiles, tiles_per_pair, grid, slot
        self.max_span = (tiles_per_cta + tiles_per_pair - 2) // tiles_per_pair + 1 + max_span_delta
        self.ws_bytes = _align_up(grid * self.max_span * slot * 4, 256)


def build_plan(nb, N, K, C, num_sms):
    """lm_build.cu build_plan: 64-point tiles, one CTA per SM at padded K >= 128, else two."""
    tpp = (N + TILE - 1) // TILE
    per_sm = 1 if padded_K(K) >= 128 else 2
    return Plan(nb * tpp, tpp, num_sms * per_sm, slot_floats(K, C))


def build_plan_tc(nb, N, K, C, num_sms, grid_wh=None):
    """lm_build_tc_host.cu build_plan_tc: 8x8-pixel tiles under the dense-grid hint, else 64 consecutive points; one CTA per SM."""
    tpp = ((grid_wh[0] + 7) // 8) * ((grid_wh[1] + 7) // 8) if grid_wh else (N + TILE - 1) // TILE
    return Plan(nb * tpp, tpp, num_sms, slot_floats(K, C))


def keyframe_plan(nw, nf, N, K, C, num_sms):
    """lm_window_key.cu keyframe_plan: tiles per window, one slot of nf frames per (CTA, span)."""
    tpw = (N + TILE - 1) // TILE
    return Plan(nw * tpw, tpw, num_sms * (1 if padded_K(K) >= 128 else 2), key_slot_floats(K, C, nf))


def part_begin(total, parts, i):
    return total * i // parts


def _begins(plan, partition=part_begin):
    return np.array([partition(plan.total_tiles, plan.grid, c) for c in range(plan.grid + 1)], dtype=np.int64)


def span_walk(plan, partition=part_begin):
    """Slots the build kernel writes: arrays (cta, span, pair), one entry per (CTA, span).  Asserts that the three roles of the
    tensor-core kernel and the SIMT kernel's walk agree on every span."""
    tpp = plan.tiles_per_pair
    beg = _begins(plan, partition)
    ctas, spans, pairs = [], [], []
    for c in range(plan.grid):
        tb, te = int(beg[c]), int(beg[c + 1])
        n = te - tb
        if n <= 0:
            continue
        b = np.arange(tb, te, dtype=np.int64) // tpp
        change = np.ones(n, dtype=bool)
        change[1:] = b[1:] != b[:-1]
        span = np.cumsum(change) - 1                               # SIMT / keyframe walk and the algebra warps' sspan
        dumps = b[np.flatnonzero(np.append(change[1:], True))]     # gather warps: dump at the next pair change and at the end
        rr0 = (tb & 0xFFFFFFFF) % tpp                              # (unsigned)t_begin % tiles_per_pair
        last = ((rr0 + np.arange(1, n + 1)) % tpp == 0)
        last[-1] = True                                            # ... || j == ntiles - 1
        flush_pairs, flush_spans = b[last], span[last]             # algebra flush(sspan) / MMA write(span) at last_of_pair
        mma_spans = np.arange(int(last.sum()))                     # the MMA warps' own counter (++span after each write)
        starts = np.flatnonzero(change)
        assert np.array_equal(flush_pairs, b[starts]), (c, "a role flushes a span the walk does not start")
        assert np.array_equal(flush_spans, span[starts]) and np.array_equal(mma_spans, span[starts]), (c, "span counters disagree")
        assert np.array_equal(dumps, b[starts]), (c, "gather hand-over out of step with the algebra warps")
        ctas.append(np.full(starts.size, c, dtype=np.int64)); spans.append(span[starts]); pairs.append(b[starts])
    return np.concatenate(ctas), np.concatenate(spans), np.concatenate(pairs)


def reduce_slots(plan, npairs, partition=part_begin, span_offset=0):
    """Slots the reduce reads: arrays (cta, span, pair).  One vector lane per pair, stepping through lm_reduce_kernel's thread-0 loop."""
    tpp, grid, total = plan.tiles_per_pair, plan.grid, plan.total_tiles
    beg = _begins(plan, partition)
    b = np.arange(npairs, dtype=np.int64)
    p0 = b * tpp
    p1 = p0 + tpp
    c0 = (p0 * grid) // total
    while True:                                                    # while (c0 + 1 < grid && part_begin(c0 + 1) <= p0) ++c0;
        m = (c0 + 1 < grid) & (beg[np.minimum(c0 + 1, grid)] <= p0)
        if not m.any():
            break
        c0 = c0 + m
    n = np.zeros(npairs, dtype=np.int64)
    alive = np.ones(npairs, dtype=bool)
    ctas, spans, pairs = [], [], []
    c = c0.copy()
    while alive.any():
        alive &= (c < grid) & (n < REDUCE_CAP)
        cc = np.minimum(c, grid - 1)
        tb, te = beg[cc], beg[cc + 1]
        alive &= tb < p1                                           # if (tb >= p1) break;
        take = alive & (tb < te) & (te > p0)                       # if (tb >= te || te <= p0) continue;
        idx = np.flatnonzero(take)
        ctas.append(c[idx]); spans.append(b[idx] - tb[idx] // tpp + span_offset); pairs.append(b[idx])
        n += take
        c = c + 1
    return np.concatenate(ctas), np.concatenate(spans), np.concatenate(pairs)


def check_partition(plan, npairs, partition_kernel=part_begin, partition_reduce=part_begin, span_offset=0):
    """Every written slot is read exactly once and by its own pair; spans stay below max_span; slots stay inside ws_bytes; no pair is
    spread over more CTAs than the reduce can list.  Returns the largest span count and CTA count per pair seen."""
    wc, ws, wb = span_walk(plan, partition_kernel)
    rc, rs, rb = reduce_slots(plan, npairs, partition_reduce, span_offset)
    assert int(ws.max()) < plan.max_span, ("span >= max_span", int(ws.max()), plan.max_span)
    wid, rid = wc * plan.max_span + ws, rc * plan.max_span + rs
    assert int(rs.min()) >= 0 and int(rs.max()) < plan.max_span, "the reduce reads a span outside the CTA's slots"
    assert (int(wid.max()) + 1) * plan.slot_floats * 4 <= plan.ws_bytes, "slot past the workspace"
    assert np.unique(wid).size == wid.size, "two spans write one slot"
    assert int(wb.min()) >= 0 and int(wb.max()) < npairs, "pair index out of range"
    per_pair = np.bincount(wb, minlength=npairs)
    assert int(per_pair.min()) >= 1, "a pair has no slot"
    assert int(per_pair.max()) <= REDUCE_CAP, ("more CTAs on one pair than the reduce lists", int(per_pair.max()))
    ow, orr = np.lexsort((wb, wid)), np.lexsort((rb, rid))
    assert np.array_equal(wid[ow], rid[orr]) and np.array_equal(wb[ow], rb[orr]), "written and read slots differ"
    return int(ws.max()) + 1, int(per_pair.max())
