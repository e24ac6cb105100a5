"""Floor type 1 (Vorbis I section 7.2.4; audio.rs:354-555): every place the library builds the curve on the device, post
layouts that each reach a named edge of those places, and a plain Python-integer walk of the decode to hold them to.
Pure Python: the CPU suite checks the walk against the oracle and that every layout reaches its edge; the GPU module runs
the layouts through each site.

Sites (lewton_b200/csrc):
  F1  k_floor1_segments + k_prologue_fused<false>: the residue entry's front stages (uniform 2048, 1024, 512, the one-pass
      256/2048 schedule, and the four-kernel path on 16-byte aligned arenas).  A bin finds its segment in a per-row bitmap
      of flagged posts plus a prefix byte per 32-bin word (kernel_prologue.cuh: k_floor1_segments, d_floor_quad_one);
      rows with a segment longer than 4096 bins take the post-shift (SHIFT) form of d_floor1_seg_y;
  F2  the same with k_prologue_fused<true>: the VQ entry;
  F3  k_chain's front half, residue entry (interleaved output, <= 8 channels, any blocksize 64..8192): a binary search
      per bin, d_floor1_y_at (floor1_eval.cuh), posts in 8 x 66-entry shared arrays;
  F4  the same, VQ entry;
  F5  k_prologue with <= 8 channels (the four-kernel path on arenas the front stages refuse, lwb_decode_packet,
      lwb_debug_packet_taps): the reference's integer DDA, d_floor1_render_segment, one lane per segment, into a byte
      curve in shared memory;
  F6  k_prologue with more than 8 channels: d_floor1_y_at, 8 channels per group.

Layouts (each constructor returns Layout objects; `edge` names the edge, which the CPU test checks each one reaches):
  1 two posts at rangebits 0, 1, 4, 15: one segment plus a flat tail or a truncation;
  2 a full table: 65 posts, every one flagged, the last below n/2 (m = 66 with the tail);
  3 the last flagged post at n/2, n/2 - 1, n/2 + 1: no tail, a one-bin tail, a segment across the end.  Post 1 of the
    last two is not a power of two: lwb_setup_create takes such lists, the header parser never makes them (every other
    layout's post 1 is 2^rangebits);
  4 an x list reaching 2^15 whose segment over bin n/2 - 1 is longer than 4096 bins;
  5 adjacent posts (adx = 1), |dy| = 255 (multiplier 1) and 252 (multiplier 4) of both signs, dy = 0, DDA segments
    with base != 0;
  6 flagged posts at bitmap word boundaries, 2 to 4 flagged posts in one 4-bin quad, a 32-bin word flagged throughout;
  7 post 64 flagged and not flagged (d_floor1_posts' flag64), unflagged posts between flagged ones;
  8 the clamp: final y at range - 1 and above it for each multiplier, and y values up to 2^24 - 1 that wrap
    render_point's u32 product."""
import numpy as np

FRONT = frozenset({"k_floor1_segments", "k_prologue_fused"})
RANGE = (256, 128, 86, 64)                 # by multiplier - 1 (audio.rs:393)

# site: (what selects it, kernels that must run, kernels that must not)
SITES = {
    "F1": ("residue entry, <= 8 channels, aligned arenas, not interleaved", FRONT, {"k_prologue", "k_chain"}),
    "F2": ("VQ entry through the four-kernel path", FRONT, {"k_prologue", "k_chain"}),
    "F3": ("residue entry, interleaved output, <= 8 channels", {"k_chain"}, FRONT | {"k_prologue"}),
    "F4": ("VQ entry, interleaved output, <= 8 channels", {"k_chain"}, FRONT | {"k_prologue"}),
    "F5": ("k_prologue, <= 8 channels: LWB_FORCE_GENERIC=1 on a residue arena off 16 bytes, lwb_debug_packet_taps",
           {"k_prologue"}, FRONT | {"k_chain"}),
    "F6": ("more than 8 channels", {"k_prologue"}, FRONT | {"k_chain"}),
}


# ---------------------------------------------------------------------------------------------------------------------
# the walk
# ---------------------------------------------------------------------------------------------------------------------
def _i32(v):
    return ((v + (1 << 31)) & 0xffffffff) - (1 << 31)


def _neighbours(xs, i):
    lo = max((j for j in range(i) if xs[j] < xs[i]), key=lambda j: xs[j])
    hi = min((j for j in range(i) if xs[j] > xs[i]), key=lambda j: xs[j])
    return lo, hi


def _predict(xs, fy, i):
    """render_point (audio.rs:354-367) of post i from its neighbours, u32 / i32 wrapping.  Returns (its product
    |dy| * (x - x0) before the u32 wrap, the prediction as i32)."""
    lo, hi = _neighbours(xs, i)
    dy = _i32(fy[hi] - fy[lo])
    prod = abs(dy) * (xs[i] - xs[lo])
    off = (prod & 0xffffffff) // (xs[hi] - xs[lo])
    return prod, _i32(fy[lo] - off if dy < 0 else fy[lo] + off)


def _step(pred, val, rng_y):
    """The un-wrapping of one coded value (audio.rs:401-429) in signed integers."""
    highroom, lowroom = rng_y - pred, pred
    room = min(highroom, lowroom) * 2
    if val <= 0:
        return pred
    if val >= room:
        return pred + val - lowroom if highroom > lowroom else pred - val + highroom - 1
    return pred + ((-val - 1 if val % 2 == 1 else val) >> 1)


def unwrap(xs, mult, y):
    """Floor-1 step 1 (audio.rs:391-435) in Python integers.  Returns the products |dy| * (x - x0) render_point forms
    (u32 in the reference: >= 2^32 wraps), the final y values before the clamp (as u32) and the step-2 flags.  Asserts
    that the signed arithmetic stays inside i32, where the reference and the oracle agree."""
    rng_y = RANGE[mult - 1]
    fy, prods, flag = [y[0], y[1]], [], [True, True] + [False] * (len(xs) - 2)
    for i in range(2, len(xs)):
        prod, pred = _predict(xs, fy, i)
        prods.append(prod)
        r = _step(pred, y[i], rng_y)
        assert all(-(1 << 31) <= v < (1 << 31) for v in (rng_y - pred, 2 * min(rng_y - pred, pred), r)), \
            "beyond the reference's i32 arithmetic"
        if y[i] > 0:
            lo, hi = _neighbours(xs, i)
            flag[lo] = flag[hi] = flag[i] = True
        fy.append(r & 0xffffffff)
    return prods, fy, flag


def render_line(x0, y0, x1, y1):
    """render_line (audio.rs:503-524): the integer DDA, bins [x0, x1)."""
    dy, adx = y1 - y0, x1 - x0
    base = abs(dy) // adx * (1 if dy >= 0 else -1)        # truncation toward zero
    sy = base - 1 if dy < 0 else base + 1
    ady = abs(dy) - abs(base) * adx
    y, err, out = y0, 0, [y0]
    for _ in range(x0 + 1, x1):
        err += ady
        if err >= adx:
            err -= adx
            y += sy
        else:
            y += base
        out.append(y)
    return out


def flagged_posts(xs, mult, y):
    """The posts step 2 draws, in x order, as (x, y * multiplier) with y clamped to range - 1 (audio.rs:431-433, 528-545):
    the first post and every flagged one."""
    _, fy, flag = unwrap(xs, mult, y)
    top = RANGE[mult - 1] - 1
    order = sorted(range(len(xs)), key=lambda i: xs[i])
    return [(xs[i], min(fy[i], top) * mult) for k, i in enumerate(order) if k == 0 or flag[i]]


def walk(xs, mult, y, n2):
    """The curve of n2 bins (curve y values, before the dB table) that step 2 renders: render_line from post to flagged
    post, a flat tail to n2 when the last flagged post is below it, truncated to n2 (audio.rs:528-550)."""
    posts = flagged_posts(xs, mult, y)
    curve = []
    for (lx, ly), (hx, hy) in zip(posts, posts[1:]):
        curve += render_line(lx, ly, hx, hy)
    hx, hy = posts[-1]
    if hx < n2:
        curve += render_line(hx, hy, n2, hy)
    return curve[:n2]


def segments(xs, mult, y, n2):
    """The segments the device draws: [(x0, y0, x1, y1)] between consecutive flagged posts, the flat tail included."""
    posts = flagged_posts(xs, mult, y)
    if posts[-1][0] < n2:
        posts.append((n2, posts[-1][1]))
    return [(a[0], a[1], b[0], b[1]) for a, b in zip(posts, posts[1:])]


# ---------------------------------------------------------------------------------------------------------------------
# post layouts
# ---------------------------------------------------------------------------------------------------------------------
class Layout:
    """One floor (multiplier, x list) and one packet's coded y values, built to reach `edge` at n2 bins."""

    def __init__(self, name, edge, mult, xs, y, n2):
        assert len(xs) == len(y) <= 65 and xs[0] == 0 and len(set(xs)) == len(xs)
        self.name, self.edge, self.mult, self.xs, self.y, self.n2 = name, edge, mult, list(xs), list(y), n2

    def walk(self, n2=None):
        return walk(self.xs, self.mult, self.y, self.n2 if n2 is None else n2)

    def segments(self, n2=None):
        return segments(self.xs, self.mult, self.y, self.n2 if n2 is None else n2)

    def __repr__(self):
        return f"{self.name}@{self.n2}"


def encode(xs, mult, targets):
    """Coded y values whose step 1 gives post i the final value targets[i], or the nearest one a nonzero coded value
    reaches (a flagged post never keeps its prediction: a target equal to it moves by one).  None: the coded value 0,
    the post left unflagged unless a later post flags it.  Posts 0 and 1 take their targets as they are."""
    rng_y = RANGE[mult - 1]
    y, fy = [targets[0], targets[1]], [targets[0], targets[1]]
    for i in range(2, len(xs)):
        _, pred = _predict(xs, fy, i)
        t = targets[i]
        if t is None:
            y.append(0)
            fy.append(pred & 0xffffffff)
            continue
        if t == pred:
            t = t + 1 if t < 200 else t - 1
        d = t - pred
        val = next((v for v in (2 * d if d > 0 else -2 * d - 1, t, rng_y - 1 - t) if v > 0 and _step(pred, v, rng_y) == t),
                   None)
        if val is None:
            val = min(range(1, 4 * rng_y), key=lambda v: abs(_step(pred, v, rng_y) - t))
        y.append(val)
        fy.append(_step(pred, val, rng_y) & 0xffffffff)
    return y


def _flagged_targets(rng, xs, mult, lo=0, hi=None):
    """Targets in [lo, hi] for every post, each one away from the post's prediction so that every post is flagged."""
    rng_y = RANGE[mult - 1]
    hi = rng_y - 1 if hi is None else hi
    t = [int(rng.integers(lo, hi + 1)), int(rng.integers(lo, hi + 1))]
    for i in range(2, len(xs)):
        _, pred = _predict(xs, t, i)
        v = int(rng.integers(lo, hi + 1))
        t.append(v if v != pred else (v + 1 if v < hi else v - 1))
    return t


def two_posts(rng, n2):
    """Layout 1: [0, 2^rangebits] at rangebits 0, 1, 4 and 15."""
    out = []
    for rb in (0, 1, 4, 15):
        mult = 1 + rb % 4
        xs = [0, 1 << rb]
        out.append(Layout(f"two_posts_rb{rb}", "tail" if (1 << rb) < n2 else "truncation", mult, xs,
                          encode(xs, mult, _flagged_targets(rng, xs, mult)), n2))
    return out


def full_table(rng, n2):
    """Layout 2: 65 posts, all flagged, the last (post 1) below n/2.  Needs n/2 >= 128."""
    if n2 < 128:
        return []
    top = min(n2 // 2, 1024)
    xs = [0, top] + [int(v) for v in rng.choice(np.arange(1, top), 63, replace=False)]
    mult = 2
    return [Layout("full_table", "m == 66", mult, xs, encode(xs, mult, _flagged_targets(rng, xs, mult)), n2)]


def end_posts(rng, n2):
    """Layout 3: post 1 (always flagged: the last flagged post) at n/2, n/2 - 1 and n/2 + 1, with 12 posts below."""
    out = []
    for d, edge in ((0, "no tail"), (-1, "one-bin tail"), (1, "segment across the end")):
        top = n2 + d
        xs = [0, top] + [int(v) for v in rng.choice(np.arange(1, top), 12, replace=False)]
        mult = 3
        out.append(Layout(f"end_at_n2{d:+d}", edge, mult, xs, encode(xs, mult, _flagged_targets(rng, xs, mult)), n2))
    return out


def long_x_list(rng, n2):
    """Layout 4: rangebits 15 (post 1 at 2^15), 20 posts below n/2 - 1 and 20 more than 4096 bins above n/2, a steep
    segment across n/2 - 1: the segment over bin n/2 - 1 spans more than 4096 bins (the post-shift form)."""
    lo = rng.choice(np.arange(1, n2 - 1), min(20, n2 - 2), replace=False)
    hi = rng.choice(np.arange(n2 + 4200, 1 << 15), 20, replace=False)
    xs = [0, 1 << 15] + [int(v) for v in rng.permutation(np.concatenate([lo, hi]))]
    mult = 1
    t = _flagged_targets(rng, xs, mult)
    below = max(range(len(xs)), key=lambda i: xs[i] if xs[i] < n2 else -1)
    above = min(range(len(xs)), key=lambda i: xs[i] if xs[i] >= n2 else 1 << 20)
    return [Layout("long_x_list", "segment > 4096 over n/2 - 1", mult, xs,
                   encode(xs, mult, _steep(t, xs, below, above, 0, 255)), n2)]


def _steep(t, xs, a, b, ya, yb):
    """Targets t with posts a and b (a coded before b or not) set to ya and yb, recomputed so every post stays flagged:
    only the values of a and b change, the others keep theirs when they differ from their new prediction."""
    t = list(t)
    t[a], t[b] = ya, yb
    for i in range(2, len(xs)):
        if i in (a, b):
            continue
        _, pred = _predict(xs, t, i)
        if t[i] == pred:
            t[i] = pred + 1 if pred < 200 else pred - 1
    return t


def steep_and_flat(rng, n2):
    """Layout 5: adjacent posts (adx = 1) with |dy| = 255 both ways (multiplier 1) and |dy| = 252 (multiplier 4, y 0 <->
    63), dy = 0 segments, and DDA segments with base = dy / adx != 0 of both signs."""
    out = []
    top = 32 if n2 < 64 else 64
    # multiplier 1: 0 at x = 10, 255 at 11, 0 at 12 (adjacent, both signs); 255 -> 0 over 7 bins (base -36); flat 40..60
    xs = [0, top, 10, 11, 12, 20, 27, 40, 60]
    t = [128, 128, 0, 255, 0, 255, 0, 90, 90]
    if top < 64:                                        # flat 27..29 instead
        xs, t = xs[:7] + [29], t[:7] + [0]
    out.append(Layout("steep_255", "|dy| = 255 at adx = 1, base != 0, dy = 0", 1, xs, encode(xs, 1, t), n2))
    # multiplier 4: 63 * 4 = 252 both ways, adjacent; 0 -> 63 over 5 bins (base 50); flat run
    xs = [0, top, 3, 4, 5, 10, 15, 20]
    t = [30, 30, 63, 0, 63, 0, 63, 63]
    out.append(Layout("steep_252", "|dy| = 252 at adx = 1, base != 0, dy = 0", 4, xs, encode(xs, 4, t), n2))
    return out


def word_boundaries(rng, n2):
    """Layout 6: flagged posts at x = 32k - 1 and 32k, two, three and four flagged posts inside one 4-bin quad, and one
    32-bin word with every bin flagged."""
    words = max(1, n2 // 32)
    full = 1 if words >= 3 else 0                       # the word flagged throughout
    xs = list(range(32 * full, 32 * full + 32))
    for k in range(1, min(words, 5)):
        xs += [32 * k - 1, 32 * k]
    if words >= 3:
        q = 32 * 2 + 8                                  # quads of word 2: 2, 3 and 4 posts
        xs += [q, q + 1, q + 5, q + 6, q + 7, q + 8, q + 9, q + 10, q + 11]
    xs = sorted(set(xs) - {0})
    top = 1 << max(xs).bit_length()
    xs = [0, top] + [x for x in xs if x < top][:63]
    mult = 2
    return [Layout("word_boundaries", "flags at word edges, in one quad, a full word", mult, xs,
                   encode(xs, mult, _flagged_targets(rng, xs, mult)), n2)]


def post64(rng, n2):
    """Layout 7: 65 posts, post 64 (the last coded) flagged and not flagged; one post in three left unflagged."""
    out = []
    top = max(64, min(n2 // 2, 2048))
    xs = [0, top] + [int(v) for v in rng.choice(np.arange(1, top), 63, replace=False)]
    mult = 3
    for on in (True, False):
        t = _flagged_targets(rng, xs, mult)
        t = [v if i < 2 or i == 64 or i % 3 else None for i, v in enumerate(t)]
        if not on:
            t[64] = None
        out.append(Layout(f"post64_{'on' if on else 'off'}", f"post 64 {'flagged' if on else 'unflagged'}", mult, xs,
                          encode(xs, mult, t), n2))
    return out


def clamp(rng, n2):
    """Layout 8: per multiplier, final y values at range - 1 and above it (posts 0 and 1 too), and, multiplier 1, coded
    values up to 2^24 - 1 whose products wrap render_point's u32 arithmetic."""
    out = []
    top = max(64, min(n2 // 2, 2048))
    for mult in (1, 2, 3, 4):
        rng_y = RANGE[mult - 1]
        xs = [0, top] + [int(v) for v in rng.choice(np.arange(1, top), 30, replace=False)]
        t = [rng_y - 1, rng_y + 7] + [rng_y - 1 if i % 3 == 0 else int(rng.integers(rng_y, 2 * rng_y)) if i % 3 == 1
                                      else int(rng.integers(0, rng_y)) for i in range(2, len(xs))]
        out.append(Layout(f"clamp_m{mult}", "final y at range - 1 and above", mult, xs, encode(xs, mult, t), n2))
    for k in range(8):              # a draw that wraps and keeps the step-2 arithmetic inside i32
        r = np.random.default_rng(int(rng.integers(1 << 30)) + k)
        xs = [0, 4096] + [int(v) for v in r.choice(np.arange(1, 4096), 40, replace=False)]
        y = [255, int(r.integers(0, 256))]
        y += [0 if r.random() < 0.3 else int(r.integers(1, 40)) if r.random() < 0.5 else int(r.integers(1 << 20, 1 << 24))
              for _ in range(len(xs) - 2)]
        try:
            prods, _, _ = unwrap(xs, 1, y)
        except AssertionError:
            continue
        if any(p >= 1 << 32 for p in prods):
            out.append(Layout("wrap", "render_point product >= 2^32", 1, xs, y, n2))
            break
    return out


CONSTRUCTORS = (two_posts, full_table, end_posts, long_x_list, steep_and_flat, word_boundaries, post64, clamp)


def layouts(n2, seed=0):
    """Every layout that can reach its edge at n2 bins."""
    rng = np.random.default_rng(seed * 8191 + n2)
    return [lay for f in CONSTRUCTORS for lay in f(rng, n2)]
