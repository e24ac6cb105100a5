"""Case generators for the row copies of k_row_copy (lewton_b200/csrc/path_chain.cuh), and the classes of row they
reach.  Pure Python: the CPU suite checks that the generators reach every class, the GPU modules run them.

k_row_copy stores a row of `nbytes` in three parts: a head of 2-byte stores up to the destination's next 16-byte
boundary (or the whole row, if it is shorter), whole 16-byte lines, and a tail of 2-byte stores.  Each line is
funnel-shifted out of the two source lines it straddles; which shift template runs depends on the phase, the source
address minus the destination address mod 16.  So a row's class is (phase, head, lines, tail), computed here from the
byte addresses mod 16 that the library gives the row:
  * a clipped chain's full output sits in scratch planes of a multiple of 8 elements that start at the PCM base's
    offset mod 16 (place_clipped_chains); so plane k of a planar chain is copied from sample `skip` of a plane at the
    base's phase, and an interleaved chain from element skip * K;
  * a host-memory batch stages its PCM in device memory from an 8-element boundary below its first chain, so there
    the phase of the caller's base does not reach the kernel: only element offsets mod 8 do;
  * a state row (lwb_streams_save / load) is 16-byte aligned on the device; the buffer side sits at the buffer's base
    plus the slot's offset plus c * len (device memory), or, in host memory, in staging that starts at the lowest
    offset of a slot with rows."""

LINE = 16


def split(dst_byte, nbytes):
    """(head, lines, tail) in bytes, lines in 16-byte lines, of a row of nbytes stored at a destination dst_byte mod 16."""
    head = min(nbytes, (LINE - dst_byte % LINE) % LINE)
    lines = (nbytes - head) // LINE
    return head, lines, nbytes - head - LINE * lines


class Row:
    """One k_row_copy row: source and destination byte addresses mod 16, its length in bytes, the element size."""

    def __init__(self, src_byte, dst_byte, nbytes, esz):
        self.esz, self.nbytes = esz, nbytes
        self.phase = (src_byte - dst_byte) % LINE
        self.to_boundary = (LINE - dst_byte % LINE) % LINE
        self.head, self.lines, self.tail = split(dst_byte, nbytes)


def classes(esz):
    """Every class a batch of rows of esz-byte elements has to reach."""
    n = LINE // esz
    want = {("phase", p) for p in range(0, LINE, esz)}
    want |= {("head", h) for h in range(n)} | {("tail", t) for t in range(n)}
    return want | {("shorter than its head",), ("one line",), ("no row",), ("long row",)}


def reached(rows, esz, empty):
    """The classes `rows` reach; empty: how many chains or slots move nothing (no row at all)."""
    got = set()
    for r in rows:
        assert r.esz == esz and r.nbytes > 0 and r.nbytes % esz == 0
        if r.lines:                      # the phase picks the shift template of the line loop
            got.add(("phase", r.phase))
        got.add(("head", r.head // esz))
        got.add(("tail", r.tail // esz))
        if r.nbytes < r.to_boundary:
            got.add(("shorter than its head",))
        if (r.head, r.lines, r.tail) == (0, 1, 0):
            got.add(("one line",))
        if r.lines >= 64:
            got.add(("long row",))
    if empty:
        got.add(("no row",))
    return got


def missing(rows, esz, empty, want=None):
    return sorted((want if want is not None else classes(esz)) - reached(rows, esz, empty))


# ---------------------------------------------------------------------------------------------------------------------
# part 1: clipped chains (output windows)
# ---------------------------------------------------------------------------------------------------------------------
LIMITS = list(range(1, 18)) + [31, 32, 33, None]      # None: to the end of the chain


def windows(n, line):
    """(skip, limit) of each chain of a batch whose chains produce n samples each: first a chain that writes `line`
    samples (one 16-byte line per row), then skip residues 0..7 reached as s, 64 * j + s and 1024 + s, every limit of
    LIMITS, and the windows that write nothing (a limit of 0, a skip past the chain) or a whole chain but its first
    samples.  Every window clips its chain, so the batch keeps its unwindowed path."""
    out = [(5, line)]
    for j in range(96):
        s = j % 8
        skip = (s, 64 * (1 + (j // 8) % 15) + s, 1024 + s)[j % 3]
        out.append((skip, LIMITS[(j * 5) % len(LIMITS)]))
    out += [(0, 0), (n + 5, None), (3, None), (n - 1, None)]
    assert all(w[0] < n for w in out[:97])
    return out


def clip(window, n):
    """(skip, written) of a chain producing n samples under window (skip, limit): window_clip of pcm_copy_plan.h."""
    skip, limit = window
    s = min(skip, n)
    return s, n - s if limit is None else min(limit, n - s)


def dst_residues(j):
    """Destination residues mod 8 of chain j's first and second plane."""
    return (3 * j + j // 8) % 8, (5 * j + 1 + j // 16) % 8


def layout(windows_, n, Ks, planar, packed, start=0):
    """[(out_offset, out_stride)] of the windowed chains (Ks: output channels of each) and the arena size in elements.
    Padded: every plane at its residue of dst_residues() past `start`, with at least 4 elements of sentinel around it.
    Packed: out_stride == written, chains back to back from `start`, no padding anywhere, so a store past a row lands
    in the next row.  (start: an element offset at a 16-byte boundary of the arena.)"""
    lay, at = [], start
    for j, (w, K) in enumerate(zip(windows_, Ks)):
        written = clip(w, n)[1]
        if packed:
            lay.append((at, written if planar else 0))
            at += K * written
            continue
        d0, d1 = dst_residues(j)
        off = at + 4 + (start + d0 - (at + 4)) % 8
        if planar:
            stride = written + 4 + (start + d1 - (off + written + 4)) % 8
            lay.append((off, stride))
            at = off + K * stride
        else:
            lay.append((off, 0))
            at = off + K * written + 4
    return lay, at + 8


def window_rows(windows_, lay, n, Ks, planar, esz, base_byte):
    """The k_row_copy rows of a windowed batch, and how many clipped chains move nothing.  Ks: output channels per
    chain; base_byte: the PCM base's byte offset mod 16 as the kernel sees it (0 for host memory)."""
    rows, empty = [], 0
    for w, (off, stride), K in zip(windows_, lay, Ks):
        skip, written = clip(w, n)
        if (skip, written) == (0, n):
            continue                     # not clipped: no row copy
        if not written:
            empty += 1
            continue
        if planar:
            rows += [Row(base_byte + skip * esz, base_byte + (off + k * stride) * esz, written * esz, esz) for k in range(K)]
        else:
            rows.append(Row(base_byte + skip * K * esz, base_byte + off * esz, written * K * esz, esz))
    return rows, empty


# ---------------------------------------------------------------------------------------------------------------------
# part 2: lwb_streams_save / lwb_streams_load
# ---------------------------------------------------------------------------------------------------------------------
def state_lengths(n1):
    """The loaded state lengths: small ones around every multiple of 4, and blocksize_1 / 2 = n1 // 2."""
    return [0, 1, 2, 3, 4, 5, 7, 8, 9, 31, 32, 33, 127, 128, n1 // 2]


def state_slots(lengths, C, gap):
    """[(offset, len)] of one slot per (residue, length) and the buffer's size in elements: four rounds over `lengths`.
    gap set: round r's slots at offsets of residue r mod 4, at least one element apart.  gap 0: each round's slots back
    to back from an offset of residue r (C * len is even for stereo, so the round's start sets the odd residues)."""
    out, at = [], 0
    for r in range(4):
        if not gap:
            at += 1 + (r - (at + 1)) % 4
        for n in lengths:
            if gap:
                at += 1 + (r - (at + 1)) % 4
            out.append((at, n))
            at += C * n
    return out, at + 4


def state_rows(slots, C, base, host, load):
    """The k_row_copy rows of a save (load False) or a load of `slots` from a buffer `base` floats past a 16-byte
    boundary, and how many slots move nothing.  The stream's state rows are 16-byte aligned."""
    used = [o for o, n in slots if n]
    lo = min(used) if used else 0
    rows, empty = [], 0
    for off, n in slots:
        if not n:
            empty += 1
            continue
        for c in range(C):
            b = ((off - lo + c * n) * 4) if host else ((base + off + c * n) * 4)
            rows.append(Row(b, 0, n * 4, 4) if load else Row(0, b, n * 4, 4))
    return rows, empty


def load_classes():
    """A load stores into the aligned state rows: every row starts on a line, so its head is always empty."""
    return classes(4) - {("head", h) for h in range(1, 4)} - {("shorter than its head",)}
