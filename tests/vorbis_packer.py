"""Synthetic Vorbis I bitstream packer -- TEST INFRASTRUCTURE for the host front end
(include/lewton_frontend.h).  There are no Vorbis files in the build image and the reference crate
cannot be built, so the tests make their own streams: random but valid setup headers (codebooks with
random complete Huffman trees, VQ lookup types 1 and 2, floor types 0 and 1, residue types 0, 1 and 2,
submaps, coupling, several modes) and audio packets whose content the packer chooses itself.  Because
the packer knows what it wrote, it knows what a correct decoder must produce: every codeword it emits
is logged as an *event* (end bit position + what it adds to which output), so the expected floor
posts / residue vectors are available for the whole packet and for any truncation of it (Vorbis I
spec sections 2-4, 7, 8; end-of-packet rules in audio.rs:82-104, :640-716).

Written from the Vorbis I specification's encoder-side view; shares no code with the C++ decoder."""
import struct

import numpy as np


class BitWriter:
    def __init__(self):
        self.bits = []

    def write(self, value, nbits):
        assert 0 <= value < (1 << nbits) or nbits == 0, (value, nbits)
        for i in range(nbits):
            self.bits.append((value >> i) & 1)

    def write_bits(self, bitlist):
        self.bits.extend(bitlist)

    def pos(self):
        return len(self.bits)

    def bytes(self):
        b = bytearray((len(self.bits) + 7) // 8)
        for i, bit in enumerate(self.bits):
            if bit:
                b[i >> 3] |= 1 << (i & 7)
        return bytes(b)


def ilog(v):
    r = 0
    while v:
        r += 1
        v >>= 1
    return r


def float32_pack(x):
    """Vorbis float32: sign | 10-bit exponent (bias 788) | 21-bit mantissa; x must be exactly representable."""
    if x == 0:
        return 0
    sign = 0x80000000 if x < 0 else 0
    m = abs(x)
    e = 0
    while m != int(m):
        m *= 2
        e -= 1
    m = int(m)
    while m >= (1 << 21):
        assert m % 2 == 0, "not representable"
        m //= 2
        e += 1
    return sign | ((e + 788) << 21) | m


def assign_codewords(lengths):
    """Vorbis canonical assignment (spec 3.2.1): each entry, in order, gets the lowest-valued free
    codeword of its length.  Returns, per entry, the list of bits in the order they are written
    (most significant codeword bit first), or None for unused entries."""
    out = [None] * len(lengths)
    available = [0] * 33           # available[d]: a free node at depth d (left-aligned in 32 bits), 0 = none
    first = True
    for i, ln in enumerate(lengths):
        if ln == 0:
            continue
        if first:
            first = False
            res = 0
            for d in range(1, ln + 1):
                available[d] = 1 << (32 - d)
        else:
            z = ln
            while z > 0 and not available[z]:
                z -= 1
            assert z > 0, "overspecified tree"
            res = available[z]
            available[z] = 0
            for d in range(ln, z, -1):
                available[d] = res + (1 << (32 - d))
        out[i] = [(res >> (31 - k)) & 1 for k in range(ln)]
    return out


def random_lengths(rng, used, max_len=12):
    """Lengths of a complete prefix code with `used` codewords (used >= 2), or [1] for used == 1."""
    if used == 1:
        return [1]
    leaves = [0]
    while len(leaves) < used:
        cand = [i for i, d in enumerate(leaves) if d < max_len]
        i = cand[int(rng.integers(0, len(cand)))]
        d = leaves.pop(i)
        leaves += [d + 1, d + 1]
    rng.shuffle(leaves)
    return [int(d) for d in leaves]


class Codebook:
    def __init__(self, rng, entries, dims, lookup_type=0, sparse_unused=0, ordered=False, max_len=12):
        self.entries, self.dims, self.lookup_type = entries, dims, lookup_type
        used = entries - sparse_unused
        lens = random_lengths(rng, used, max_len)
        if ordered:
            lens = sorted(lens)
            sparse_unused = 0
            self.entries = entries = used
        self.ordered = ordered
        self.lengths = [0] * entries
        slots = sorted(rng.permutation(entries)[:used].tolist())
        for s, ln in zip(slots, lens):
            self.lengths[s] = ln
        self.codes = assign_codewords(self.lengths)
        self.used_entries = [i for i, ln in enumerate(self.lengths) if ln]
        self.vq = None
        if lookup_type:
            self.minimum = float(rng.integers(-8, 4)) / 4.0
            self.delta = float(rng.integers(1, 9)) / 8.0
            self.value_bits = int(rng.integers(2, 7))
            self.sequence_p = bool(rng.integers(0, 2))
            if lookup_type == 1:
                lv = 0
                while (lv + 1) ** dims <= entries:
                    lv += 1
                self.lookup_values = lv
            else:
                self.lookup_values = entries * dims
            self.multiplicands = rng.integers(0, 1 << self.value_bits, self.lookup_values).tolist()
            self.set_values(self.minimum, self.delta, self.sequence_p)

    def set_values(self, minimum, delta, sequence_p):
        """Value mapping of a VQ book (minimum, delta: exactly representable as Vorbis float32) and its vq table."""
        self.minimum, self.delta, self.sequence_p = minimum, delta, sequence_p
        entries, dims = self.entries, self.dims
        vq = np.zeros((entries, dims), np.float32)
        mn, dl = np.float32(self.minimum), np.float32(self.delta)
        for e in range(entries):
            last = np.float32(0)
            div = 1
            for k in range(dims):
                if self.lookup_type == 1:
                    mo = (e // div) % self.lookup_values
                    div *= self.lookup_values
                else:
                    mo = e * dims + k
                v = np.float32(np.float32(np.float32(self.multiplicands[mo]) * dl) + mn) + last
                v = np.float32(v)
                if self.sequence_p:
                    last = v
                vq[e, k] = v
        self.vq = vq

    def write_header(self, w):
        w.write(0x564342, 24)
        w.write(self.dims, 16)
        w.write(self.entries, 24)
        if self.ordered:
            w.write(1, 1)
            cur = 0
            ln = self.lengths[0]
            w.write(ln - 1, 5)
            while cur < self.entries:
                number = sum(1 for x in self.lengths[cur:] if x == ln)
                # lengths are sorted: entries of this length are contiguous
                w.write(number, ilog(self.entries - cur))
                cur += number
                ln += 1
        else:
            w.write(0, 1)
            sparse = any(x == 0 for x in self.lengths)
            w.write(int(sparse), 1)
            for ln in self.lengths:
                if sparse:
                    w.write(int(ln > 0), 1)
                    if ln:
                        w.write(ln - 1, 5)
                else:
                    w.write(ln - 1, 5)
        w.write(self.lookup_type, 4)
        if self.lookup_type:
            w.write(float32_pack(self.minimum), 32)
            w.write(float32_pack(self.delta), 32)
            w.write(self.value_bits - 1, 4)
            w.write(int(self.sequence_p), 1)
            for m in self.multiplicands:
                w.write(m, self.value_bits)

    def emit(self, w, entry):
        w.write_bits(self.codes[entry])

    def random_entry(self, rng):
        return self.used_entries[int(rng.integers(0, len(self.used_entries)))]


class Floor1:
    def __init__(self, rng, books, n_books_scalar, rangebits=None, multiplier=None):
        """books: list of Codebook; scalar books (lookup 0 is fine) are picked among the first n_books_scalar."""
        self.multiplier = int(multiplier or rng.integers(1, 5))
        self.rangebits = int(rangebits or rng.integers(6, 11))
        n_part = int(rng.integers(1, 6))
        n_class = int(rng.integers(1, 4))
        self.partition_class = rng.integers(0, n_class, n_part).tolist()
        n_class = max(self.partition_class) + 1
        self.class_dims = rng.integers(1, 5, n_class).tolist()
        self.class_sub = rng.integers(0, 3, n_class).tolist()
        self.master = []
        self.sub_books = []
        for c in range(n_class):
            sub = self.class_sub[c]
            nsb = 1 << sub
            # the master book's entry selects one sub book per dimension (successive cbits-wide digits)
            cands = list(range(n_books_scalar))
            self.master.append(int(cands[int(rng.integers(0, len(cands)))]) if sub else 0)
            sb = []
            for _ in range(nsb):
                sb.append(-1 if rng.random() < 0.2 else int(rng.integers(0, n_books_scalar)))
            self.sub_books.append(sb)
        count = 2 + sum(self.class_dims[c] for c in self.partition_class)
        xs = rng.permutation(np.arange(1, 1 << self.rangebits))[: count - 2].tolist()
        self.x_list = [0, 1 << self.rangebits] + [int(x) for x in xs]

    def write_header(self, w):
        w.write(1, 16)
        w.write(len(self.partition_class), 5)
        for c in self.partition_class:
            w.write(c, 4)
        for c in range(len(self.class_dims)):
            w.write(self.class_dims[c] - 1, 3)
            w.write(self.class_sub[c], 2)
            if self.class_sub[c]:
                w.write(self.master[c], 8)
            for b in self.sub_books[c]:
                w.write(b + 1, 8)
        w.write(self.multiplier - 1, 2)
        w.write(self.rangebits, 4)
        for x in self.x_list[2:]:
            w.write(x, self.rangebits)

    def write_packet(self, w, rng, books, unused=False):
        """Returns the y list the decoder must produce (None = unused)."""
        if unused:
            w.write(0, 1)
            return None
        w.write(1, 1)
        rng_y = [256, 128, 86, 64][self.multiplier - 1]
        b = ilog(rng_y - 1)
        y = [int(rng.integers(0, rng_y)), int(rng.integers(0, rng_y))]
        w.write(y[0], b)
        w.write(y[1], b)
        for c in self.partition_class:
            cdim, cbits = self.class_dims[c], self.class_sub[c]
            csub = (1 << cbits) - 1
            cval = 0
            if cbits:
                mb = books[self.master[c]]
                cval = mb.random_entry(rng)
                # the decoder indexes sub_books with successive cbits-wide digits of cval
                mb.emit(w, cval)
            for _ in range(cdim):
                book = self.sub_books[c][cval & csub]
                cval >>= cbits
                if book >= 0:
                    e = books[book].random_entry(rng)
                    books[book].emit(w, e)
                    y.append(e)
                else:
                    y.append(0)
        return y


class Floor0:
    def __init__(self, rng, books, vq_book_ids):
        self.order = int(rng.integers(2, 12))
        self.rate = int(rng.choice([8000, 22050, 44100, 48000]))
        self.bark_map_size = int(rng.integers(16, 300))
        self.amplitude_bits = int(rng.integers(4, 9))
        self.amplitude_offset = int(rng.integers(20, 120))
        nb = int(rng.integers(1, 4))
        self.book_list = [int(vq_book_ids[int(rng.integers(0, len(vq_book_ids)))]) for _ in range(nb)]

    def write_header(self, w):
        w.write(0, 16)
        w.write(self.order, 8)
        w.write(self.rate, 16)
        w.write(self.bark_map_size, 16)
        w.write(self.amplitude_bits, 6)
        w.write(self.amplitude_offset, 8)
        w.write(len(self.book_list) - 1, 4)
        for b in self.book_list:
            w.write(b, 8)

    def write_packet(self, w, rng, books, unused=False):
        """Returns (amplitude, [vq rows]) or None."""
        if unused:
            w.write(0, self.amplitude_bits)
            return None
        amp = int(rng.integers(1, 1 << self.amplitude_bits))
        w.write(amp, self.amplitude_bits)
        bn = int(rng.integers(0, len(self.book_list)))
        w.write(bn, ilog(len(self.book_list)))
        book = books[self.book_list[bn]]
        rows = []
        got = 0
        while got < self.order:
            e = book.random_entry(rng)
            book.emit(w, e)
            rows.append(book.vq[e].copy())
            got += book.dims
        return amp, rows


class Residue:
    def __init__(self, rng, books, vq_book_ids, class_book_ids, n2_long, rtype=None, cascade_p=0.5):
        self.type = int(rng.integers(0, 3)) if rtype is None else rtype
        self.classifications = int(rng.integers(1, 5))
        # classbook: dims = classwords per codeword, entries >= classifications ** dims, all used
        while True:
            cands = [i for i in class_book_ids if books[i].entries >= self.classifications ** books[i].dims]
            if cands:
                break
            self.classifications -= 1
        self.classbook = int(cands[int(rng.integers(0, len(cands)))])
        self.partition_size = int(rng.choice([8, 16, 32]))
        self.begin = int(rng.integers(0, 3)) * self.partition_size
        self.end = int(n2_long * (2 if self.type == 2 else 1) * rng.choice([0.5, 1.0, 1.5]))
        self.end = max(self.end, self.begin)
        self.cascade = []
        self.books = []
        for _ in range(self.classifications):
            # bit 7 is never read back by lewton (ResidueBook::read_book reads 7 books)
            c = sum(1 << q for q in range(7) if rng.random() < cascade_p) if rng.random() < 0.8 else 0
            row = []
            for p in range(8):
                if c & (1 << p):
                    cands = [b for b in vq_book_ids if self.partition_size % books[b].dims == 0]
                    row.append(int(cands[int(rng.integers(0, len(cands)))]))
                else:
                    row.append(None)
            self.cascade.append(c)
            self.books.append(row)

    def write_header(self, w):
        w.write(self.type, 16)
        w.write(self.begin, 24)
        w.write(self.end, 24)
        w.write(self.partition_size - 1, 24)
        w.write(self.classifications - 1, 6)
        w.write(self.classbook, 8)
        for c in self.cascade:
            w.write(c & 7, 3)
            if c >> 3:
                w.write(1, 1)
                w.write(c >> 3, 5)
            else:
                w.write(0, 1)
        for c, row in zip(self.cascade, self.books):
            for p in range(8):
                if c & (1 << p):
                    w.write(row[p], 8)

    def write_packet(self, w, rng, books, blocksize, dnd, events):
        """Emit the residue of one submap.  dnd: do-not-decode flag per channel of the submap.
        Appends events (end_bit, channel_in_submap, index array, value array)."""
        ch = len(dnd)
        if self.type == 2:
            if all(dnd):
                return
            self._write_inner(w, rng, books, blocksize * ch, [False], events, interleave=ch)
        else:
            self._write_inner(w, rng, books, blocksize, dnd, events, interleave=0)

    def _write_inner(self, w, rng, books, blocksize, dnd, events, interleave):
        actual = blocksize // 2
        lb, le = min(self.begin, actual), min(self.end, actual)
        cb = books[self.classbook]
        cpc = cb.dims
        n_to_read = le - lb
        parts = n_to_read // self.partition_size
        if n_to_read == 0:
            return
        ch = len(dnd)
        cls = np.zeros((ch, parts + cpc), np.int64)
        for pas in range(8):
            pc = 0
            while pc < parts:
                if pas == 0:
                    for j in range(ch):
                        if dnd[j]:
                            continue
                        digits = rng.integers(0, self.classifications, cpc)
                        entry = 0
                        for d in digits:
                            entry = entry * self.classifications + int(d)
                        cb.emit(w, entry)
                        cls[j, pc: pc + cpc] = digits
                        events.append((w.pos(), None, None, None))
                for _ in range(cpc):
                    if pc >= parts:
                        break
                    for j in range(ch):
                        if dnd[j]:
                            continue
                        book_id = self.books[int(cls[j, pc])][pas] if self.cascade[int(cls[j, pc])] & (1 << pas) else None
                        if book_id is None:
                            continue
                        book = books[book_id]
                        offs = lb + pc * self.partition_size
                        if self.type == 0:
                            step = self.partition_size // book.dims
                            for i in range(step):
                                e = book.random_entry(rng)
                                book.emit(w, e)
                                idx = offs + i + np.arange(book.dims) * step
                                self._event(events, w.pos(), j, idx, book.vq[e], interleave, actual)
                        else:
                            i = 0
                            while i < self.partition_size:
                                e = book.random_entry(rng)
                                book.emit(w, e)
                                idx = offs + i + np.arange(book.dims)
                                self._event(events, w.pos(), j, idx, book.vq[e], interleave, actual)
                                i += book.dims
                    pc += 1

    @staticmethod
    def _event(events, pos, j, idx, vals, interleave, actual):
        keep = idx < actual
        idx, vals = idx[keep], vals[keep]
        if interleave:
            # residue 2: one interleaved vector, element i belongs to channel i % ch at index i // ch
            for c in range(interleave):
                sel = (idx % interleave) == c
                if sel.any():
                    events.append((pos, c, idx[sel] // interleave, vals[sel]))
            if not len(idx):
                events.append((pos, None, None, None))
        else:
            events.append((pos, j, idx, vals))


class StreamSpec:
    """A random valid set of headers.  channels, blocksizes (log2), and knobs for which features appear."""

    def __init__(self, rng, channels=2, bs0=8, bs1=11, floor0=False, n_modes=None, sample_rate=44100, residue_types=None,
                 cascade_p=0.5):
        self.rng = rng
        self.channels, self.bs0, self.bs1, self.sample_rate = channels, bs0, bs1, sample_rate
        # codebooks: scalar books first (floor-1 values / class words), then VQ books
        self.books = []
        n_scalar = int(rng.integers(3, 6))
        for i in range(n_scalar):
            entries = int(rng.choice([4, 16, 27, 64, 81, 256]))
            self.books.append(Codebook(rng, entries, int(rng.integers(1, 4)), 0, ordered=(i == 1)))
        self.books.append(Codebook(rng, 1, 1, 0))                     # single-entry book (1-bit code)
        self.n_scalar = len(self.books)
        vq_ids = []
        for i in range(int(rng.integers(3, 6))):
            dims = int(rng.choice([1, 2, 4, 8]))
            lt = int(rng.integers(1, 3))
            entries = int(rng.choice([8, 16, 81, 100]))
            unused = int(rng.integers(0, entries // 4)) if rng.random() < 0.5 else 0
            self.books.append(Codebook(rng, entries, dims, lt, sparse_unused=unused))
            vq_ids.append(len(self.books) - 1)
        self.vq_ids = vq_ids
        class_ids = list(range(n_scalar))
        self.floors = []
        for i in range(int(rng.integers(1, 4))):
            if floor0 and i == 0:
                self.floors.append(Floor0(rng, self.books, vq_ids))
            else:
                self.floors.append(Floor1(rng, self.books, self.n_scalar))
        self.residues = []
        n2_long = (1 << bs1) // 2
        rts = residue_types or [None] * int(rng.integers(1, 4))
        for rt in rts:
            self.residues.append(Residue(rng, self.books, vq_ids, class_ids, n2_long, rt, cascade_p))
        self.mappings = []
        for _ in range(int(rng.integers(1, 3))):
            submaps = int(rng.integers(1, min(3, channels) + 1))
            steps = []
            if channels > 1:
                for _ in range(int(rng.integers(0, channels + 1))):
                    m, a = rng.choice(channels, 2, replace=False)
                    steps.append((int(m), int(a)))
            mux = rng.integers(0, submaps, channels).tolist() if submaps > 1 else [0] * channels
            self.mappings.append({"submaps": submaps, "coupling": steps, "mux": mux,
                                  "floors": rng.integers(0, len(self.floors), submaps).tolist(),
                                  "residues": rng.integers(0, len(self.residues), submaps).tolist()})
        n_modes = n_modes or int(rng.integers(2, 5))
        self.modes = [(0, int(rng.integers(0, len(self.mappings)))), (1, int(rng.integers(0, len(self.mappings))))]
        while len(self.modes) < n_modes:
            self.modes.append((int(rng.integers(0, 2)), int(rng.integers(0, len(self.mappings)))))
        self.vendor = "lewton_b200 synthetic packer"
        self.comments = [("TITLE", "synthetic"), ("ARTIST", "packer éè")]

    # ---- headers ---------------------------------------------------------------------------------
    def ident_packet(self):
        return (b"\x01vorbis" + struct.pack("<IBIiiiB", 0, self.channels, self.sample_rate, 0, 128000, 0,
                                            self.bs0 | (self.bs1 << 4)) + b"\x01")

    def comment_packet(self, extra_raw=()):
        v = self.vendor.encode()
        out = b"\x03vorbis" + struct.pack("<I", len(v)) + v
        items = [("%s=%s" % kv).encode() for kv in self.comments] + list(extra_raw)
        out += struct.pack("<I", len(items))
        for it in items:
            out += struct.pack("<I", len(it)) + it
        return out + b"\x01"

    def setup_packet(self):
        w = BitWriter()
        for b in b"\x05vorbis":
            w.write(b, 8)
        w.write(len(self.books) - 1, 8)
        for b in self.books:
            b.write_header(w)
        w.write(0, 6)
        w.write(0, 16)
        w.write(len(self.floors) - 1, 6)
        for f in self.floors:
            f.write_header(w)
        w.write(len(self.residues) - 1, 6)
        for r in self.residues:
            r.write_header(w)
        w.write(len(self.mappings) - 1, 6)
        cil = ilog(self.channels - 1)
        for m in self.mappings:
            w.write(0, 16)
            if m["submaps"] > 1:
                w.write(1, 1)
                w.write(m["submaps"] - 1, 4)
            else:
                w.write(0, 1)
            if m["coupling"]:
                w.write(1, 1)
                w.write(len(m["coupling"]) - 1, 8)
                for mag, ang in m["coupling"]:
                    w.write(mag, cil)
                    w.write(ang, cil)
            else:
                w.write(0, 1)
            w.write(0, 2)
            if m["submaps"] > 1:
                for c in range(self.channels):
                    w.write(m["mux"][c], 4)
            for s in range(m["submaps"]):
                w.write(0, 8)
                w.write(m["floors"][s], 8)
                w.write(m["residues"][s], 8)
        w.write(len(self.modes) - 1, 6)
        for bf, mp in self.modes:
            w.write(bf, 1)
            w.write(0, 16)
            w.write(0, 16)
            w.write(mp, 8)
        w.write(1, 1)
        return w.bytes()

    # ---- audio packets ---------------------------------------------------------------------------
    def audio_packet(self, mode, prev_flag=1, next_flag=1, p_unused=0.15):
        """Returns (bytes, info).  info: mode, flags, n, floors (per channel: None | ('one', y) |
        ('zero', amp, rows)), floor_end_bits (per channel), events (residue), header_bits."""
        rng = self.rng
        w = BitWriter()
        w.write(0, 1)
        w.write(mode, ilog(len(self.modes) - 1))
        bf, mp_i = self.modes[mode]
        n = 1 << (self.bs1 if bf else self.bs0)
        if bf:
            w.write(prev_flag, 1)
            w.write(next_flag, 1)
        header_bits = w.pos()
        mp = self.mappings[mp_i]
        floors, floor_ends = [], []
        for c in range(self.channels):
            fl = self.floors[mp["floors"][mp["mux"][c]]]
            unused = rng.random() < p_unused
            r = fl.write_packet(w, rng, self.books, unused)
            if r is None:
                floors.append(None)
            elif isinstance(fl, Floor1):
                floors.append(("one", r))
            else:
                floors.append(("zero", r[0], r[1], fl))
            floor_ends.append(w.pos())
        no_res = [f is None for f in floors]
        for mag, ang in mp["coupling"]:
            if not (no_res[mag] and no_res[ang]):
                no_res[mag] = no_res[ang] = False
        events = []
        for s in range(mp["submaps"]):
            chans = [c for c in range(self.channels) if mp["mux"][c] == s]
            dnd = [no_res[c] for c in chans]
            sub_events = []
            self.residues[mp["residues"][s]].write_packet(w, rng, self.books, n, dnd, sub_events)
            for pos, j, idx, vals in sub_events:
                events.append((pos, None if j is None else chans[j], idx, vals))
        info = {"mode": mode, "blockflag": bf, "prev": prev_flag if bf else 1, "next": next_flag if bf else 1, "n": n,
                "floors": floors, "floor_ends": floor_ends, "events": events, "header_bits": header_bits,
                "total_bits": w.pos(), "mapping": mp}
        return w.bytes(), info

    def expected(self, info, nbytes=None):
        """What a correct decoder produces from the first nbytes of the packet (None = all of it):
        (floor list per channel as in info['floors'] with None for unused, residue [channels][n/2] f32)."""
        limit = info["total_bits"] if nbytes is None else nbytes * 8
        n2 = info["n"] // 2
        floors = []
        for c in range(self.channels):
            floors.append(info["floors"][c] if info["floor_ends"][c] <= limit else None)
        # a truncated floor makes that channel unused; the coupling propagation is re-evaluated by the decoder,
        # but nothing after the cut can be read anyway
        res = np.zeros((self.channels, n2), np.float32)
        if all(e <= limit for e in info["floor_ends"]):
            for pos, c, idx, vals in info["events"]:
                if pos > limit:
                    break
                if c is None:
                    continue
                res[c, idx] = res[c, idx] + vals.astype(np.float32)
        return floors, res


# ---- Ogg pages -------------------------------------------------------------------------------------
def _crc_table():
    t = []
    for i in range(256):
        r = i << 24
        for _ in range(8):
            r = ((r << 1) ^ 0x04C11DB7) & 0xFFFFFFFF if r & 0x80000000 else (r << 1) & 0xFFFFFFFF
        t.append(r)
    return t


_CRC = _crc_table()


def ogg_crc(data):
    c = 0
    for b in data:
        c = ((c << 8) & 0xFFFFFFFF) ^ _CRC[((c >> 24) ^ b) & 0xFF]
    return c


def ogg_page(serial, seq, absgp, packets_segments, bos=False, eos=False, continued=False):
    """packets_segments: list of (bytes, complete) -- payload pieces on this page; complete=False means
    the packet continues on the next page (its last lacing value is 255)."""
    lacing = bytearray()
    body = bytearray()
    for data, complete in packets_segments:
        ln = len(data)
        full, rem = divmod(ln, 255)
        lacing += bytes([255] * full)
        if complete:
            lacing.append(rem)
        else:
            assert rem == 0, "a continued packet must fill whole segments"
        body += data
    assert len(lacing) <= 255
    htype = (1 if continued else 0) | (2 if bos else 0) | (4 if eos else 0)
    hdr = b"OggS" + struct.pack("<BBQIII", 0, htype, absgp, serial, seq, 0) + bytes([len(lacing)]) + bytes(lacing)
    page = bytearray(hdr + body)
    crc = ogg_crc(page)
    page[22:26] = struct.pack("<I", crc)
    return bytes(page)


def ogg_stream(serial, header_packets, audio_packets, absgps, packets_per_page=3, split_large=True):
    """Pages: ident alone (bos), comment+setup, then audio packets_per_page per page with the given
    granule position per page (absgps: one per audio page).  Packets longer than 255*255 bytes are not
    produced by the packer; a packet that does not fit the remaining lacing of a page is continued."""
    pages = []
    seq = 0
    pages.append(ogg_page(serial, seq, 0, [(header_packets[0], True)], bos=True))
    seq += 1
    # comment + setup may be large: split over continued pages
    pending = [header_packets[1], header_packets[2]]
    segs, room, continued = [], 255, False
    for pk in pending:
        data = pk
        while True:
            need = len(data) // 255 + 1
            if need <= room:
                segs.append((data, True))
                room -= need
                break
            take = room * 255
            segs.append((data[:take], False))
            pages.append(ogg_page(serial, seq, 0, segs, continued=continued))
            seq += 1
            data = data[take:]
            segs, room, continued = [], 255, True
    if segs:
        pages.append(ogg_page(serial, seq, 0, segs, continued=continued))
        seq += 1
    groups = [audio_packets[i: i + packets_per_page] for i in range(0, len(audio_packets), packets_per_page)]
    assert len(absgps) == len(groups)
    for gi, grp in enumerate(groups):
        pages.append(ogg_page(serial, seq, absgps[gi], [(p, True) for p in grp], eos=(gi == len(groups) - 1)))
        seq += 1
    return b"".join(pages)
