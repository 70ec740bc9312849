"""Row builders for the exact node2vec step (euler_b200/csrc/walk.cu): graphs whose biased rows make the sequential f32
prefix of CompactWeightedCollection::Init round, tie, change binade, sit at zero or go subnormal on purpose, plus a numpy
replay of that prefix that counts those events.  Plain numpy: the CPU tests check the generators with it, the GPU tests
build their graphs with it.

Every hub row H comes with a start node A that lists H (weight 1) and, with weight 0, a chosen subset of H's neighbors.
Zero weights are never drawn, so every walker started at A is at H after step 0, and at step 1 H's row is biased against
A's list: the subset keeps its weight (shared), A itself is divided by p, every other entry by q (BuildWeights)."""
import numpy as np

# walk.cu's launch thresholds
K_PREF_HEAD = 768       # kPrefHead: elements summed serially before the first parallel iteration
K_WALK_BIG = 512        # rows longer than this: k_walk_prefix_cta<256>
K_WALK_HUGE = 16384     # rows longer than this: k_walk_prefix_cta<1024>

# row lengths at every boundary of the step kernels: warp chunks, warp / CTA-256 / CTA-1024, the serial head, one
# CTA-256 and one CTA-1024 iteration after it, and a long row (the 600K-entry one has a test of its own)
BOUNDARY_LENGTHS = [1, 32, 33, 511, 512, 513, 767, 768, 769, 768 + 1024 - 1, 768 + 1024, 768 + 1024 + 1, 16384, 16385,
                    768 + 4096 - 1, 768 + 4096, 768 + 4096 + 1, 70_000]


# ------------------------------------------------------------------------------------------------------ BuildWeights
def build_weights_literal(cn, w, pn, parent_id, p, q):
    """tf_euler/kernels/random_walk_op.cc:140-168 as written: the two-pointer merge with int64 compares."""
    w = np.array(w, np.float32)
    p, q = np.float32(p), np.float32(q)
    j = k = 0
    cn, pn = [int(x) for x in np.asarray(cn, np.int64)], [int(x) for x in np.asarray(pn, np.int64)]
    while j < len(cn) and k < len(pn):
        if cn[j] < pn[k]:
            w[j] = w[j] / q if cn[j] != parent_id else w[j] / p
            j += 1
        elif cn[j] == pn[k]:
            j += 1
            k += 1
        else:
            k += 1
    while j < len(cn):
        w[j] = w[j] / q if cn[j] != parent_id else w[j] / p
        j += 1
    return w


def build_weights(cn, w, pn, parent_id, p, q):
    """The same merge for lists sorted in int64 order, as the per-element rule the parallel kernels use: the m-th copy of v
    in the child list is shared iff the parent list holds more than m copies of v."""
    cn, pn = np.asarray(cn, np.int64), np.asarray(pn, np.int64)
    w = np.asarray(w, np.float32)
    first = np.searchsorted(cn, cn, side="left")
    m = np.arange(len(cn)) - first
    cnt = np.searchsorted(pn, cn, side="right") - np.searchsorted(pn, cn, side="left")
    shared = m < cnt
    div = np.where(cn == np.int64(parent_id), np.float32(p), np.float32(q)).astype(np.float32)
    return np.where(shared, w, w / div).astype(np.float32)


def stored_weights(cum):
    """What both the device and the oracle read for one row: cum[j] - cum[j-1] in f32 (cum[-1] = 0)."""
    cum = np.asarray(cum, np.float32)
    return np.diff(cum, prepend=np.float32(0)).astype(np.float32)


# ------------------------------------------------------------------------------------------------- prefix events
def prefix(v):
    """S_k = fl(S_{k-1} + v_k) left to right in f32 (np.add.accumulate is a sequential loop)."""
    return np.add.accumulate(np.asarray(v, np.float32), dtype=np.float32)


def _event_masks(v):
    """Per addition k: S_k, S_{k-1}, and masks of the inexact ones and of the four kinds of event below."""
    v = np.asarray(v, np.float32)
    S = prefix(v)
    prev = np.concatenate([np.zeros(1, np.float32), S[:-1]])
    exact = prev.astype(np.float64) + v.astype(np.float64)   # exact whenever a tie is possible (exponents within 29 binades)
    lo, hi = np.nextafter(S, np.float32(-np.inf)), np.nextafter(S, np.float32(np.inf))
    S64 = S.astype(np.float64)
    e_prev, e_S, e_v = np.frexp(prev)[1], np.frexp(S)[1], np.frexp(v)[1]
    normal = prev >= np.finfo(np.float32).tiny
    return S, prev, dict(
        inexact=exact != S64,
        tie=(exact == (lo.astype(np.float64) + S64) / 2) | (exact == (S64 + hi.astype(np.float64)) / 2),
        binade=(prev > 0) & (e_S > e_prev),
        above=(v > 0) & normal & (e_v > e_prev),
        tiny_S=(v > 0) & ~normal)


def prefix_events(v, start=K_PREF_HEAD):
    """Counts, over the additions k >= start, the cases block_exact_prefix must leave its integer fast path for, and the
    plain inexact ones.  tie: the exact S_{k-1} + v_k is the midpoint of two f32s; binade: S changes exponent; above: v_k's
    exponent exceeds S_{k-1}'s; tiny_S: S_{k-1} is 0 or subnormal while v_k > 0."""
    v = np.asarray(v, np.float32)
    S, prev, ev = _event_masks(v)
    sel = np.arange(len(v)) >= start
    z = np.concatenate([[0], (v[start:] == 0).astype(np.int8), [0]]) if len(v) > start else np.zeros(2, np.int8)
    edges = np.flatnonzero(np.diff(z))
    out = {k: int((sel & m).sum()) for k, m in ev.items()}
    out.update(n=int(sel.sum()), zero_run=int((edges[1::2] - edges[0::2]).max()) if len(edges) else 0,
               S_start=float(prev[start]) if len(v) > start else float(S[-1]) if len(v) else 0.0,
               total=float(S[-1]) if len(v) else 0.0)
    return out


def exception_positions(v):
    """Positions k where block_exact_prefix cannot take v_k as an integer increment in S_{k-1}'s binade: exact ties,
    binade steps, addends above S's binade, and nonzero addends to S = 0 or subnormal (every weight here is >= 0)."""
    _, _, ev = _event_masks(v)
    return np.flatnonzero(ev["tie"] | ev["binade"] | ev["above"] | ev["tiny_S"])


def prefix_iterations(v, threads, serial=96, elems=4):
    """Iterations of the total pass of block_exact_prefix<threads> over the row: one for the serial head, then per
    iteration either a whole stretch of threads * elems elements (no exception in it) or everything up to the first
    exception plus `serial` elements summed one by one."""
    n, ch = len(v), threads * elems
    if n == 0:
        return 0
    exc = exception_positions(v)
    pos, it = min(n, K_PREF_HEAD), 1
    while pos < n:
        n_it = min(ch, n - pos)
        i = np.searchsorted(exc, pos)
        f = exc[i] - pos if i < len(exc) else n_it
        pos += n_it if f >= n_it else min(f + serial, n_it)
        it += 1
    return it


# ---------------------------------------------------------------------------------------------------- families
# Each returns (w, shared_mask, p, q): the stored weights of a hub row of n entries (exact f32 running sums unless said
# otherwise) and which entries the start node lists.
def tie_heavy(n, rng):
    """Integers around m = 0.97 * 2^24 / n, a quarter of them shared and odd, q = 0.5: the biased S passes 2^24 (ulp 2)
    while the stored cum_w stays below it, so every shared odd weight after that is an exact tie."""
    m = max(4, int(0.97 * 2 ** 24 / max(n, 1)))
    w = rng.randint(m // 2, m + m // 2, size=n).astype(np.int64)
    shared = rng.rand(n) < 0.25
    w[shared] |= 1
    return w.astype(np.float32), shared, 2.0, 0.5


def random_rounding(n, rng):
    """Integers 1..k (k = 1000, less on long rows so that cum_w stays below 2^24), q = 3, p = 0.7: nearly every biased
    weight and every addition is inexact."""
    k = max(2, min(1000, int(0.9 * 2 ** 25 / max(n, 1))))
    return (1 + rng.randint(0, k, size=n)).astype(np.float32), rng.rand(n) < 0.25, 0.7, 3.0


def zero_runs(n, rng):
    """Integer weights with runs of 4096 .. 6000 zeros after the head."""
    w, shared, p, q = random_rounding(n, rng)
    pos = K_PREF_HEAD + 200
    while pos + 4096 < n:
        ln = int(rng.randint(4096, 6001))
        w[pos:pos + ln] = 0
        pos += ln + int(rng.randint(300, 3000))
    return w, shared, p, q


def zero_head(n, rng, nz=1200):
    """The first nz >= 1000 weights are 0: S = 0 when the parallel part starts."""
    w, shared, p, q = random_rounding(n, rng)
    w[:nz] = 0
    return w, shared, p, q


def all_zero(n, rng):
    """Every weight 0: the total is 0 and RandomSelect falls through to the last entry."""
    return np.zeros(n, np.float32), rng.rand(n) < 0.25, 0.7, 3.0


def wide_exponent(n, rng, jumps=10):
    """Weights from 2^-40 up to 2^20.  The head holds weights of 2^-40 .. 2^-25; after it, weights with exponents from
    -40 to 12 below the running sum's, and `jumps` evenly spaced weights 4 binades above the running sum (so above the
    biased sum too) that carry it up to 2^20.  The stored weights are the f32 differences of the running sum: entries far
    below its ulp are stored as 0, the others rounded to its ulp."""
    at = set(np.linspace(K_PREF_HEAD + 20, n - 1, jumps).astype(int).tolist()) if n > K_PREF_HEAD + 20 else set()
    w = np.zeros(n, np.float32)
    S = np.float32(0)
    for k in range(n):
        eS = int(np.frexp(S)[1]) - 1 if S > 0 else -40
        if k in at:
            e = eS + 4
        elif k >= K_PREF_HEAD:
            e = rng.uniform(-40, max(-40, eS - 12))
        else:
            e = rng.uniform(-40, -25)
        w[k] = np.float32(np.exp2(np.floor(min(e, 20))) * (1 + rng.rand()))
        S = np.float32(S + w[k])
    return stored_weights(prefix(w)), rng.rand(n) < 0.25, 0.7, 3.0


def subnormal(n, rng):
    """Integer multiples of 2^-149 (1..max, with the whole row's cum_w still subnormal, about 1e-39): S never leaves the
    subnormal range, q = 3 rounds every unshared one."""
    k = max(1, int(4_000_000 / max(n, 1)))
    w = ((1 + rng.randint(0, k, size=n)) * np.float64(2.0 ** -149)).astype(np.float32)
    return w, rng.rand(n) < 0.25, 0.7, 3.0


FAMILIES = dict(tie_heavy=tie_heavy, random_rounding=random_rounding, zero_runs=zero_runs, zero_head=zero_head,
                all_zero=all_zero, wide_exponent=wide_exponent, subnormal=subnormal)


# -------------------------------------------------------------------------------------------------------- graphs
class HubGraph:
    """T = 1 graph in CSR arrays (the dict graphs.random_graph returns) built from hub rows.  add_hub() adds a hub H, its
    start node A and, for H's neighbors that have no row yet, rows [H, two of H's neighbors] with small integer weights;
    walkers started at A reach H at step 0."""

    def __init__(self, seed=0):
        self.rng = np.random.RandomState(seed)
        self.blocks = []        # (ids int64[m], deg int64[m], nbr int64[sum deg], stored w f32[sum deg])
        self.hubs = []          # dict(hub, start, n, nbr, w, pn)

    def ids(self):
        return np.concatenate([b[0] for b in self.blocks]) if self.blocks else np.zeros(0, np.int64)

    def add_row(self, nid, nbr, w):
        nbr = np.asarray(nbr, np.int64)
        self.blocks.append((np.asarray([nid], np.int64), np.asarray([len(nbr)], np.int64), nbr, np.asarray(w, np.float32)))

    def add_hub(self, hub, start, nbr, w, shared, extra_parent=(), leaf_rows=True):
        """nbr: H's neighbor list (int64, stored as given); w: its stored weights; shared: mask of the entries A lists with
        weight 0; extra_parent: more zero-weight entries of A's list.  A's list is kept in int64 order."""
        nbr = np.asarray(nbr, np.int64)
        pn = np.sort(np.concatenate([[np.int64(hub)], nbr[shared], np.asarray(extra_parent, np.int64)]))
        pw = np.zeros(len(pn), np.float32)
        pw[np.flatnonzero(pn == np.int64(hub))[0]] = 1
        self.add_row(hub, nbr, w)
        self.add_row(start, pn, pw)
        self.hubs.append(dict(hub=int(hub), start=int(start), n=len(nbr), nbr=nbr, w=np.asarray(w, np.float32), pn=pn))
        if leaf_rows and len(nbr):
            leaves = np.setdiff1d(np.unique(nbr), self.ids())
            m = len(leaves)
            rows = np.stack([np.full(m, np.int64(hub)), self.rng.choice(nbr, m), self.rng.choice(nbr, m)], 1)
            rows.sort(axis=1)
            self.blocks.append((leaves, np.full(m, 3, np.int64), rows.reshape(-1),
                                (1 + self.rng.randint(0, 9, size=3 * m)).astype(np.float32)))

    def build(self, sort_u64=False):
        """sort_u64: store every row in uint64 order (ids >= 2^63 then come last) instead of as given."""
        ids = self.ids()
        assert len(np.unique(ids)) == len(ids), "a node has two rows"
        deg = np.concatenate([b[1] for b in self.blocks])
        nbr = np.concatenate([b[2] for b in self.blocks])
        w = np.concatenate([b[3] for b in self.blocks])
        grp_ptr = np.zeros(len(ids) + 1, np.int64)
        grp_ptr[1:] = np.cumsum(deg)
        row = np.repeat(np.arange(len(ids)), deg)
        if sort_u64:
            o = np.lexsort((nbr.view(np.uint64), row))
            nbr, w = nbr[o], w[o]
        cum_w = np.empty(len(w), np.float32)
        for b, e in zip(grp_ptr[:-1], grp_ptr[1:]):
            if e - b > 3:
                cum_w[b:e] = prefix(w[b:e])
        pos = np.arange(len(w)) - grp_ptr[row]
        small = (deg <= 3)[row]           # the many leaf rows: the same f32 sums, all rows at once
        for k in range(3):
            j = np.flatnonzero(small & (pos == k))
            cum_w[j] = w[j] if k == 0 else cum_w[j - 1] + w[j]
        assert np.array_equal(stored_weights_rows(cum_w, grp_ptr), w), "stored weights are not exact f32 differences"
        grp_cum = np.where(deg > 0, cum_w[np.maximum(grp_ptr[1:] - 1, 0)] if len(w) else 0, 0).astype(np.float32)
        return dict(ids=ids.view(np.uint64), node_type=np.zeros(len(ids), np.int32), node_w=np.ones(len(ids), np.float32),
                    T=1, grp_ptr=grp_ptr, nbr=nbr.view(np.uint64), w=w, cum_w=cum_w, grp_cum=grp_cum, feat=None,
                    n_node_types=1)

    @staticmethod
    def step1_row(h, p, q):
        """H's biased row at step 1 of a walker started at A (parent = A, parent list = A's list)."""
        return build_weights(h["nbr"], h["w"], h["pn"], h["start"], p, q)


def stored_weights_rows(cum_w, grp_ptr):
    """stored_weights() of every row of a CSR at once"""
    w = np.diff(cum_w, prepend=np.float32(0)).astype(np.float32)
    first = grp_ptr[:-1][np.diff(grp_ptr) > 0]
    w[first] = cum_w[first]
    return w


def hub_neighbors(n, rng, lo):
    """n neighbor ids for a hub, sorted in int64 order: drawn with repeats (multi-edges) from max(8, n // 3) ids starting
    at lo."""
    pool = max(8, n // 3)
    return np.sort(lo + rng.randint(0, pool, size=n).astype(np.int64))


# ------------------------------------------------------------------------------------------------ walker classes
def walker_classes(deg, cap_v):
    """k_walk_plan's rules for one step: deg[i] = length of walker i's list (0 = dead).  Live walkers take V space in
    walker order; the ones whose cumulative degree fits in cap_v are 'small' (<= 512), 'big' (<= 16384) or 'huge', the rest
    'ovf' (the self-contained warp path).  Returns one label per walker ('dead' for deg 0)."""
    deg = np.asarray(deg, np.int64)
    ke = np.cumsum(deg)                       # dead walkers add 0
    out = np.full(len(deg), "dead", dtype=object)
    live = deg > 0
    fits = live & (ke <= cap_v)
    out[fits & (deg <= K_WALK_BIG)] = "small"
    out[fits & (deg > K_WALK_BIG) & (deg <= K_WALK_HUGE)] = "big"
    out[fits & (deg > K_WALK_HUGE)] = "huge"
    out[live & ~fits] = "ovf"
    return out


# ----------------------------------------------------------------------------------------------- the rows walked
# row lengths of each family: past the serial head, in the CTA-256 and the CTA-1024 kernels
FAMILY_LENGTHS = dict(tie_heavy=[14_000, 20_000, 70_000], random_rounding=[2_000, 20_000, 70_000],
                      zero_runs=[20_000, 70_000], zero_head=[5_000, 20_000], all_zero=[513, 3_000, 20_000],
                      wide_exponent=[20_000, 70_000], subnormal=[2_000, 20_000])


def family_row(family, n):
    """(w, shared, p, q) of one family at length n, seeded by both"""
    return FAMILIES[family](n, np.random.RandomState(n * 7 + sorted(FAMILIES).index(family)))


def check_events(family, w, v):
    """Asserts the events `family` is built to cause on the stored row w and its biased row v, past the serial head."""
    ev = prefix_events(v)
    nz = w[K_PREF_HEAD:][w[K_PREF_HEAD:] > 0]
    if family == "tie_heavy":
        assert ev["tie"] >= 1000 and ev["binade"] >= 2, ev
    elif family == "random_rounding":
        assert ev["inexact"] >= 0.4 * ev["n"], ev
    elif family == "zero_runs":
        assert ev["zero_run"] >= 4096 and ev["inexact"] > 0, ev
    elif family == "zero_head":
        assert (w[:1000] == 0).all() and ev["S_start"] == 0 and ev["tiny_S"] >= 1 and ev["total"] > 0, ev
    elif family == "all_zero":
        assert not w.any() and ev["total"] == 0, ev
    elif family == "wide_exponent":
        assert ev["above"] >= 5 and ev["inexact"] >= 1000, ev
        assert nz.min() <= 2.0 ** -30 and nz.max() >= 2.0 ** 18, (nz.min(), nz.max())
    elif family == "subnormal":
        assert 0 < ev["total"] < np.finfo(np.float32).tiny and ev["tiny_S"] == (v[K_PREF_HEAD:] > 0).sum(), ev
        assert ((v != w) & (v.astype(np.float64) * 3 != w)).any()   # the division by q rounded some of them
    else:
        raise KeyError(family)
    return ev


def hub_graph(rows, seed=0, id0=1_000_000_000, **kw):
    """HubGraph with one hub per (w, shared): hub k at id0 + 2k, its start node at id0 + 2k + 1, neighbors drawn from a
    pool at (k + 1) * 10^7 (multi-edges included)."""
    hg = HubGraph(seed)
    for k, (w, shared) in enumerate(rows):
        nbr = hub_neighbors(len(w), hg.rng, (k + 1) * 10 ** 7)
        hg.add_hub(id0 + 2 * k, id0 + 2 * k + 1, nbr, w, shared, **kw)
    return hg
