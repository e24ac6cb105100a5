"""Blocksize tables a caller may pass in lwb_setup_desc.tables[2] instead of the generated ones, as the setup takes them
(dicts like lewton_b200.generate_tables) and as the oracle takes them (oracle.Tables.from_arrays).

A Rust binding passes the crate's cached_bs_derived (header_cached.rs:34-40), evaluated by whatever libm is behind it, so
every kernel must read the caller's a, b, c and window -- never a table of its own.  The generated tables hide a kernel
that does not: a[0] == 1.0 and a[1] == -0.0 exactly, the bs-13 window slope ends in entries that round to 1.0f, and with
blocksize_0 == blocksize_1 both tables are bit-identical.  The sets here do not:

  f64        the header_cached.rs:43-99 expressions evaluated in float64 and rounded once: a libm that rounds
             differently.  An array that comes out identical to the generated one gets a few entries moved by 1 ULP.
  scrambled  every a, b, c and window entry drawn independently with a random sign, among them exact +-0, +-1.0 and
             subnormals; bitrev stays compute_bitreverse(bs), the only one the crate makes (and the setup accepts).
  split      blocksize_0 == blocksize_1 with a canonical and a scrambled table, either way round: a kernel that reads
             the other blockflag's table shows.
"""
import numpy as np

import lewton_b200 as L

ARRAYS = ("a", "b", "c", "window")

# per blocksize, how many entries of (a, b, c, window) the float64 evaluation rounds differently from lwb_tables_generate.
# lwb_tables_generate calls the host libm's sinf / cosf on f32 arguments, so these counts belong to that libm (measured
# with glibc's): another libm, or another glibc whose sinf / cosf round differently, changes them without any change to
# the project's code.
F64_DIFFERS = {
    6: (15, 8, 6, 15),
    7: (32, 16, 10, 33),
    8: (59, 31, 21, 75),
    9: (120, 64, 41, 138),
    10: (235, 124, 87, 263),
    11: (476, 226, 174, 520),
    12: (972, 454, 345, 1098),
    13: (1953, 928, 674, 2135),
}


def canonical(bs):
    return L.generate_tables(bs)


def f64_raw(bs):
    """header_cached.rs:43-99 in float64, each entry rounded once to float32; bitrev canonical."""
    n = 1 << bs
    h = n // 2
    x = np.arange(h, dtype=np.float64)
    inner = np.sin(0.5 * np.pi * (x + 0.5) / h)
    window = np.sin(0.5 * np.pi * inner * inner)
    k = np.arange(n // 4, dtype=np.float64)
    ka, kb = k * 4.0 * np.pi / n, (2 * k + 1) * 0.5 * np.pi / n
    a = np.empty(h)
    a[0::2], a[1::2] = np.cos(ka), -np.sin(ka)
    b = np.empty(h)
    b[0::2], b[1::2] = np.cos(kb) * 0.5, np.sin(kb) * 0.5
    k8 = np.arange(n // 8, dtype=np.float64)
    kc = (2 * k8 + 1) * 2.0 * np.pi / n
    c = np.empty(n // 4)
    c[0::2], c[1::2] = np.cos(kc), -np.sin(kc)
    out = {nm: v.astype(np.float32) for nm, v in zip(ARRAYS, (a, b, c, window))}
    out["bitrev"] = canonical(bs)["bitrev"]
    return out


def differing(t, ref):
    """(a, b, c, window): how many entries of t differ in bits from ref."""
    return tuple(int(np.count_nonzero(t[k].view(np.uint32) != ref[k].view(np.uint32))) for k in ARRAYS)


def f64(bs):
    """f64_raw, with every array that equals the generated one moved by 1 ULP at three entries."""
    t, ref = f64_raw(bs), canonical(bs)
    for k in ARRAYS:
        if np.array_equal(t[k].view(np.uint32), ref[k].view(np.uint32)):
            for i in (0, len(t[k]) // 3, len(t[k]) - 1):
                t[k][i] = np.nextafter(t[k][i], np.float32(2))
    return t


# in every array, at random places: +0, -0, 1.0, -1.0 and three subnormals (the least, a middling and the greatest)
SPECIAL = np.array([0.0, -0.0, 1.0, -1.0, 1e-45, -1.5e-39, 1.1754942e-38], np.float32)


def scrambled(bs, seed=0):
    """Every a, b, c and window entry independent with a random sign: magnitudes in [0.25, 1), about 3 % each of 0 and
    1.0, and SPECIAL.  The same (bs, seed) gives the same tables."""
    rng = np.random.default_rng(1000 * bs + seed)
    t = {}
    for k in ARRAYS:
        size = len(canonical(bs)[k])
        v = rng.uniform(0.25, 1.0, size).astype(np.float32)
        pick = rng.random(size)
        v[pick < 0.03] = 0.0
        v[(pick >= 0.03) & (pick < 0.06)] = 1.0
        v *= rng.choice(np.array([-1, 1], np.float32), size)
        v[rng.choice(size, len(SPECIAL), replace=False)] = SPECIAL
        t[k] = v
    t["bitrev"] = canonical(bs)["bitrev"]
    return t


def table_set(name, bs0, bs1):
    """The setup's two tables for set `name`: "canonical", "f64", "scrambled", "split_bs1" (canonical bs0 table,
    scrambled bs1 table) or "split_bs0" (the other way round).  f64 and scrambled give equal tables for equal
    blocksizes, as a binding does."""
    if name == "canonical":
        return [canonical(bs0), canonical(bs1)]
    if name == "f64":
        return [f64(bs0), f64(bs1)]
    if name == "scrambled":
        return [scrambled(bs0), scrambled(bs1)]
    if name == "split_bs1":
        return [canonical(bs0), scrambled(bs1)]
    if name == "split_bs0":
        return [scrambled(bs0), canonical(bs1)]
    raise ValueError(name)


def oracle_pair(oracle, tabs):
    """The oracle's (t0, t1) of a setup's two table dicts."""
    return tuple(oracle.Tables.from_arrays(int(np.log2(len(t["a"]) * 2)), *(t[k] for k in ARRAYS + ("bitrev",))) for t in tabs)
