"""Python mirror of the host-side tiling of tc_conv_kernel (kernels_tc.cu): pick_row_tile, pick_bn / pick_bn_fill, the work-item count, and
the persistent schedule -- CTA b runs work items b, b + grid, ...; the producer and the MMA warpgroups carry one ring position
(STAGES slots) across all of a CTA's tiles, and the consumers park each tile's accumulators in slot (local tile index % PARKS).
Tests use it to know which schedules a shape produces without a GPU."""

SMS = 132          # H100 SXM: the production grid is min(work items, SMs)
STAGES = 4         # TMA ring depth of every tc_conv_kernel instantiation
ROWS = 128         # output pixels per tile


def pick_row_tile(n, gh, gw, rows=ROWS):
    """Images per 128-row tile (kernels_tc.cu pick_row_tile's Nt), or None when the batch has no tile."""
    t = row_tile(n, gh, gw, rows)
    return None if t is None else t[0]


def row_tile(n, gh, gw, rows=ROWS):
    """(Nt, Ht, Wt): a tile is Nt images x Ht rows x Wt columns of the row grid gh x gw, or None."""
    p = gh * gw
    if gw > rows or rows % gw:
        return None
    if p >= rows:
        ht = rows // gw
        return (1, ht, gw) if p % rows == 0 and gh % ht == 0 else None
    if rows % p or n % (rows // p):
        return None
    return rows // p, gh, gw


def pick_bn(oc):
    return 128 if oc % 128 == 0 else 64 if oc % 64 == 0 else 0


def pick_bn_fill(oc, m_tiles_x_phases, sms=SMS):
    bn = pick_bn(oc)
    while bn > 64 and m_tiles_x_phases * (oc // bn) < sms:
        bn //= 2
    return bn


def parks(bn):
    """Accumulator park slots of a tile width (TcSmem::PARKS)."""
    return 1 if bn >= 128 else 2


def geometry(kind, n, h, w, c, o, k, s, p, bn=None):
    """Work decomposition of one tc_conv_kernel launch.  kind: "fprop" (conv forward, 1x1 dense included), "dgrad" (4x4 s2 p1 input
    gradient in phase form: dy [n, h/2, w/2, o] -> dx [n, h, w, c]), "ps" (the same onto c <= 4 channels as one 3x3 conv over 2x2 output
    blocks), "wmn" (dense input gradient: [n, c] x the [c][o] weight).  bn None: the production choice (pick_bn_fill).
    Returns a dict of the TcConvParams fields that set the schedule, or None when the shape has no tensor-core tile."""
    if kind in ("fprop", "wmn"):
        gh, gw = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        taps, chunks, oc, phases = k * k, c // 64, o, 1
    else:
        gh, gw = h // 2, w // 2
        taps, chunks, phases = (9, o // 64, 1) if kind == "ps" else (4, o // 64, 4)
        oc = c
    t = row_tile(n, gh, gw)
    if t is None:
        return None
    tiles_m = n * gh * gw // ROWS
    if kind == "ps":
        bn, tiles_n = 16, 1
    else:
        bn = pick_bn_fill(oc, tiles_m * phases) if bn is None else bn
        tiles_n = oc // bn
    return dict(Nt=t[0], Ht=t[1], Wt=t[2], tiles_m=tiles_m, tiles_n=tiles_n, phases=phases, bn=bn, num_kb=taps * chunks,
                tiles=tiles_m * tiles_n * phases, oc=oc)


def grid_size(tiles, max_ctas=0, sms=SMS):
    return min(tiles, max_ctas if max_ctas > 0 else sms)


def cta_tiles(tiles, grid, b):
    """The work items CTA b runs, in order."""
    return list(range(b, tiles, grid))


def ring_slot_at_tile_start(local_index, num_kb):
    """Ring slot of the first K-block of a CTA's local_index-th tile: the ring position runs on across tiles."""
    return (local_index * num_kb) % STAGES
