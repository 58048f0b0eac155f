"""Window operators with an order-sensitive combine against a direct fold of every key's items in arrival order.

The programs of tests/cpp/ordered_programs.cu (registered at run time, as an application registers its functors) fold a polynomial
hash: (h1, q1) o (h2, q2) = (h1 (q2 + 1) + h2, (q1 + 1)(q2 + 1) - 1) with wrapping unsigned arithmetic. It is associative and not
commutative, so a kernel that folds a pane out of arrival order, combines a right child before its left sibling or walks a window
that wraps the leaf ring tail-first gets a different value, and modular integer arithmetic lets the windows be compared bit for bit.
The windows that fire, their ids and result timestamps come from the oracle (oracle/oracle.py) run on the same filtered stream with a
sum payload; the hash of window g of a key is computed from prefix hashes of the key's surviving items, arrival ranks
[g * slide, g * slide + win) (time-based: its panes' items in (pane, arrival) order).

A census -- a host model of the update kernels' control flow with the constants of wfb_kernels.cuh / wfb_lib.cu -- states which
branches each case reaches (bucket path with multi-key buckets and chunks, tiny-pane warp fold, in-kernel evaluation, eager levels
above the staged siblings, ring wrap, full-sort light and heavy keys). Every case asserts the regimes it is there for, so a case that
stops reaching its branch after a tuning change fails instead of passing without testing it.

CPU (-m "not gpu"): the program compiles, its host comb / lift agree with the numpy model, the direct fold in sum mode equals the
oracle's windows, and every GPU case reaches its regimes. GPU: the windows of every case, Reduce_GPU, and the slot sort at exactly
2^24 keys."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "windflow_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "cpp", "ordered_programs.cu")
SO = os.path.join(ROOT, "tests", "cpp", "ordered_programs.so")
NVCC = ["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr", "--expt-extended-lambda",
        "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-Xcompiler", "-fPIC", "-shared", "-diag-suppress", "186"]
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")

TUPLE64 = np.dtype([("key", "<u8"), ("id", "<u8"), ("ivalue", "<i8"), ("fvalue", "<f8"), ("pad", "<u8", (4,))])
KEY16 = np.dtype([("key", "<u8"), ("a", "<u4"), ("b", "<u4")])
RES_DTYPE = {24: np.dtype([("key", "<u8"), ("id", "<u8"), ("h", "<u4"), ("q", "<u4")]),
             32: np.dtype([("key", "<u8"), ("id", "<u8"), ("h", "<u8"), ("q", "<u8")]),
             48: np.dtype([("key", KEY16), ("id", "<u8"), ("h", "<u8"), ("q", "<u8"), ("pad", "<u8")])}
WORD = {24: np.uint32, 32: np.uint64, 48: np.uint64}
M = 0x5851F42D4C957F2D  # the multiplier (odd), the programs' params_t
MIX = (np.uint64(0x9E3779B97F4A7C15), np.uint64(0xC2B2AE3D27D4EB4F), np.uint64(0x165667B19E3779F9))


# ---------------------------------------------------------------------------------------------------------------------------------
# the test programs
# ---------------------------------------------------------------------------------------------------------------------------------
def _compile():
    from windflow_b200 import build
    build.build()
    hdrs = [os.path.join(CSRC, h) for h in ("wfb_kernels.cuh", "wfb_keys.cuh", "wfb_launch.cuh", "wfb_programs.cuh", "wfb_ptx.cuh")] + \
        [os.path.join(ROOT, "include", "wfb200.h"), SRC]
    if os.path.exists(SO) and all(os.path.getmtime(SO) > os.path.getmtime(h) for h in hdrs):
        return
    subprocess.check_call(NVCC + ["-o", SO, SRC, "-L" + os.path.join(ROOT, "windflow_b200"), "-lwfb200",
                                  "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"])


_ord = None


def _ordlib():
    """The test programs' shared object, loaded after libwfb200.so so that it binds the same library instance."""
    global _ord
    if _ord is None:
        _compile()
        from windflow_b200 import _lib
        _lib.lib()
        L = C.CDLL(SO)
        for r in (24, 32, 48):
            getattr(L, f"ord_register_{r}").restype = C.c_int
        vp, u64 = C.c_void_p, C.c_uint64
        L.ord_comb_host.argtypes = [C.c_int, u64, vp, vp, vp, vp, vp, vp, u64, C.c_int]
        L.ord_comb_host.restype = C.c_int
        L.ord_lift_host.argtypes = [C.c_int, u64, vp, u64, vp, vp, vp]
        L.ord_lift_host.restype = C.c_int
        _ord = L
    return _ord


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def progs(wfb):
    """Program id of every record size, with its result dtype registered in ops.RESULT_DTYPE for the module's duration."""
    L = _ordlib()
    ids = {r: getattr(L, f"ord_register_{r}")() for r in (24, 32, 48)}
    assert all(i >= 6 for i in ids.values()), ids
    for r, i in ids.items():
        wfb.RESULT_DTYPE[i], wfb.TUPLE_DTYPE[i] = RES_DTYPE[r], TUPLE64
    yield ids
    for i in ids.values():
        wfb.RESULT_DTYPE.pop(i, None); wfb.TUPLE_DTYPE.pop(i, None)


# ---------------------------------------------------------------------------------------------------------------------------------
# numpy model and direct fold
# ---------------------------------------------------------------------------------------------------------------------------------
def _bits(W):
    return 8 * np.dtype(W).itemsize


def np_comb(h1, q1, h2, q2, W):
    one = W(1)
    with np.errstate(over="ignore"):
        return (h1 * (q2 + one) + h2).astype(W), ((q1 + one) * (q2 + one) - one).astype(W)


def key16_word(keys):
    """pad[0] of a tuple of the 48-byte program: the a / b halves of its 16-byte key, a function of `key`."""
    with np.errstate(over="ignore"):
        return (np.asarray(keys, dtype=np.uint64) * np.uint64(0xD6E8FEB86659FD93)) ^ np.uint64(0x0123456789ABCDEF)


def np_lift_h(t, rec):
    k1 = t["pad"][:, 0] if rec == 48 else np.zeros(len(t), dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = ((t["id"] + np.uint64(1)) * MIX[0]) ^ (t["key"] * MIX[1]) ^ (k1 * MIX[2])
        x ^= x >> np.uint64(29)
        x |= np.uint64(1)
    return x.astype(WORD[rec])


def keep_mask(t):
    return t["id"] % np.uint64(7) != np.uint64(3)


def _powers(base, count, W):
    a = np.full(count, base, dtype=W)
    a[0] = 1
    with np.errstate(over="ignore"):
        return np.multiply.accumulate(a, dtype=W)


def hash_ranges(h, a, b, W):
    """Fold of h[a:b] for every (a, b): H = A_b - A_a * M^(b-a) with prefix hashes A_s = sum_{j<s} h_j M^(s-1-j), and q = M^(b-a) - 1."""
    mod = 1 << _bits(W)
    Mw = M % mod
    N = len(h)
    pw, ipw = _powers(Mw, N + 1, W), _powers(pow(Mw, -1, mod), N + 1, W)
    with np.errstate(over="ignore"):
        G = np.zeros(N + 1, dtype=W)
        G[1:] = np.cumsum(h.astype(W) * ipw[:N], dtype=W)
        A = np.zeros(N + 1, dtype=W)
        A[1:] = pw[:N] * G[1:]
        L = b - a
        return (A[b] - A[a] * pw[L]).astype(W), (pw[L] - W(1)).astype(W)


def cb_ranges(keys, rkeys, rids, win, slide):
    """Count-based windows (rkeys, rids) over the items `keys` (arrival order): the permutation sorting the items by key (stable) and
    every window's range [a, b) in it (arrival ranks [g * slide, g * slide + win) of the key)."""
    order = np.argsort(keys, kind="stable")
    sk = keys[order]
    uk, start, cnt = np.unique(sk, return_index=True, return_counts=True)
    ki = np.searchsorted(uk, rkeys)
    assert np.all(uk[ki] == rkeys)
    a = start[ki] + rids.astype(np.int64) * slide
    b = a + win
    assert np.all(b <= start[ki] + cnt[ki]), "a window past the key's items"
    return order, a, b


def tb_ranges(keys, ts, rkeys, rids, win, slide, pane):
    """Time-based windows over the items: the permutation sorting them by (key, pane) (stable: arrival order inside a pane) and the
    range of every window, the panes [g * slide, g * slide + win) / pane of its key."""
    pn = (ts // np.uint64(pane)).astype(np.uint64)
    order = np.lexsort((pn, keys))
    comp = (keys[order].astype(np.uint64) << np.uint64(32)) | pn[order]
    base = rkeys.astype(np.uint64) << np.uint64(32)
    lo = (rids.astype(np.uint64) * np.uint64(slide)) // np.uint64(pane)
    hi = (rids.astype(np.uint64) * np.uint64(slide) + np.uint64(win)) // np.uint64(pane)
    return order, np.searchsorted(comp, base | lo), np.searchsorted(comp, base | hi)


def _lift_res(t):
    """The oracle's input: survivors lifted with a sum payload (isum = id)."""
    from oracle import oracle as O
    r = np.zeros(len(t), dtype=O.RES)
    r["key"], r["isum"] = t["key"], t["id"].astype(np.int64)
    return r


def make_tuples(keys, first_id, rec):
    t = np.zeros(len(keys), dtype=TUPLE64)
    t["key"] = keys
    t["id"] = np.arange(first_id, first_id + len(keys), dtype=np.uint64)
    t["ivalue"] = t["id"].astype(np.int64) * 3 + 1
    if rec == 48:
        t["pad"][:, 0] = key16_word(t["key"])
    return t


# ---------------------------------------------------------------------------------------------------------------------------------
# census: host model of the count-based update's control flow (constants of wfb_kernels.cuh / wfb_lib.cu)
# ---------------------------------------------------------------------------------------------------------------------------------
BK_REC_BYTES, BK_THREADS, BK_KEYS, OSW_BITS, LIGHT_MAX = 16384, 128, 64, 10, 256


class Geometry:
    def __init__(self, win, slide, nb, cap, rec):
        self.win, self.slide, self.nb, self.cap, self.rec = win, slide, nb, cap, rec
        self.pane = math.gcd(win, slide)
        self.B = (nb - 1) * slide + win
        self.bp, self.wp, self.sp = self.B // self.pane, win // self.pane, slide // self.pane
        n, lg = 1, 0
        while n < self.bp + min(self.bp, 32):  # wfb_ffat_create: ring of n leaves, at least min(bp, 32) spare
            n <<= 1; lg += 1
        self.n, self.logn = n, lg
        self.defer_items = (n - self.bp + 1) * self.pane
        bits = 0
        while (1 << bits) < cap:
            bits += 1
        self.shift = bits - OSW_BITS if bits > OSW_BITS else 0  # ffat_derive_paths
        self.buckets = (1 << self.shift) <= BK_KEYS and self.pane < (1 << 32)
        self.IT = min(8, max(1, BK_REC_BYTES // (BK_THREADS * rec)))  # bk_items_per_thread
        self.CAP = BK_THREADS * self.IT
        self.sibl = 8 if rec <= 32 else (4 if rec <= 48 else (2 if rec <= 128 else 1))  # BK_SIBL
        fits = self.buckets and 2 * n * rec <= (32 << 10)
        pays = n <= 2 * max(1, lg) * self.sp * nb
        self.lazy = fits and pays


def _triggers(g, c0, c1):
    """Counts in (c0, c1] at which a group fires: B + k * slide * Nb."""
    G = g.slide * g.nb
    k = 0 if c0 < g.B else (c0 - g.B) // G + 1
    out = []
    while g.B + k * G <= c1:
        out.append((k, g.B + k * G)); k += 1
    return out


def census(g, calls):
    """Regimes reached by the slots of each call (survivors in arrival order): a dict tag -> count."""
    tags = {}

    def tag(name, k=1):
        tags[name] = tags.get(name, 0) + k
    cnt = {}
    panes_max = 0
    tag("lazy" if g.lazy else "eager")
    tag("bucket_path" if g.buckets else "full_sort")
    for slots in calls:
        slots = np.asarray(slots, dtype=np.int64)
        if len(slots) == 0:
            continue
        fired = []  # (gwid of the group's first window)
        if g.buckets:
            order = np.argsort(slots >> g.shift, kind="stable")
            ss = slots[order]
            bks, bstart = np.unique(ss >> g.shift, return_index=True)
            bend = list(bstart[1:]) + [len(ss)]
            for bk, s0, s1 in zip(bks, bstart, bend):
                lst = ss[s0:s1]
                ks_all, m_all = np.unique(lst, return_counts=True)
                tags["max_keys_per_bucket"] = max(tags.get("max_keys_per_bucket", 0), len(ks_all))
                left = dict(zip(ks_all.tolist(), m_all.tolist()))
                if len(lst) > g.CAP:
                    tag("multichunk_bucket")
                paths, rounds = {}, {}
                for ci, c0i in enumerate(range(0, len(lst), g.CAP)):
                    ks, ms = np.unique(lst[c0i:c0i + g.CAP], return_counts=True)
                    info = []
                    nseg = 0
                    for k, a in zip(ks.tolist(), ms.tolist()):
                        c = cnt.get(k, 0)
                        cp = c % g.pane
                        first = min(a, g.pane - cp)
                        nseg += 1 + (a - first + g.pane - 1) // g.pane
                        info.append((k, a, c, cp, first))
                    warp_fold = nseg > BK_THREADS
                    path = "warp" if warp_fold else "thread"
                    if warp_fold:
                        tag("warp_fold")
                        if len(ks) >= 2:
                            tag("warp_fold_multikey")
                    for k, a, c, cp, first in info:
                        paths.setdefault(k, set()).add(path)
                        if ci > 0 and cp != 0:
                            tag("open_pane_at_chunk")
                        if warp_fold and a > first and (first % 32) != 0:
                            tag("warp_subrange_split")  # a pane boundary inside a group of 32 staged records
                        c1 = c + a
                        if c1 // g.pane > c // g.pane and not g.lazy and g.logn > g.sibl:
                            tag(f"eager_above_sibl_{path}")
                        for gi, t in _triggers(g, c, c1):
                            u = t - c  # 1-based index of the triggering item among the key's items of the chunk
                            rem = left[k] - u
                            if rem >= g.defer_items:
                                tag(f"inkernel_{path}")
                                if path == "thread":
                                    j = 0 if u <= first else 1 + (u - first - 1) // g.pane
                                    key = (ci, (k - (bk << g.shift)) >> 5, j)
                                    rounds[key] = rounds.get(key, 0) + 1
                            else:
                                tag("deferred_lazy" if g.lazy else "deferred")
                            fired.append(gi * g.nb)
                        left[k] -= a
                        cnt[k] = c1
                for v in rounds.values():
                    if v >= 2:
                        tag("inkernel_thread_same_round")
                for ps in paths.values():
                    if len(ps) == 2:
                        tag("key_warp_and_thread")
        else:
            ks, ms = np.unique(slots, return_counts=True)
            for k, m in zip(ks.tolist(), ms.tolist()):
                c = cnt.get(k, 0)
                heavy = m > LIGHT_MAX
                path = "update" if heavy else "lanes"
                tag(path)
                for gi, t in _triggers(g, c, c + m):
                    if m - (t - c) >= g.defer_items:
                        tag(f"inkernel_{path}")
                    else:
                        tag("deferred")
                    fired.append(gi * g.nb)
                if heavy:  # k_ffat_update: warp takes of min(32, items left, room in the open pane)
                    j, cc = 0, c
                    while j < m:
                        room = g.pane - cc % g.pane
                        take = min(32, m - j, room)
                        if take < 32 and take == room and take < m - j:
                            tag("short_take_at_pane")
                        j += take; cc += take
                cnt[k] = c + m
        for gw in fired:
            for i in range(g.nb):
                if ((gw + i) * g.sp) % g.n + g.wp > g.n:
                    tag("window_wraps_ring")
    if cnt:
        panes_max = max(cnt.values()) // g.pane
    if panes_max >= 2 * g.n:
        tag("ring_wrapped_twice")
    return tags


def assert_regimes(tags, expect):
    missing = []
    for e in expect:
        name, least = e if isinstance(e, tuple) else (e, 1)
        if tags.get(name, 0) < least:
            missing.append(e)
    assert not missing, f"the case no longer reaches {missing}; census: {tags}"


# ---------------------------------------------------------------------------------------------------------------------------------
# count-based cases
# ---------------------------------------------------------------------------------------------------------------------------------
class Case:
    def __init__(self, name, rec, win, slide, nb, cap, nkeys, calls, batch, expect, dense=True, keys="uniform", pipelined=False,
                 move=False, seed=1, census=True):
        self.name, self.rec, self.win, self.slide, self.nb, self.cap = name, rec, win, slide, nb, cap
        self.nkeys, self.calls, self.batch, self.expect, self.dense, self.keys = nkeys, calls, batch, expect, dense, keys
        self.pipelined, self.move, self.seed, self.census = pipelined, move, seed, census

    def stream(self):
        """Per call, the list of its batches (tuples, ts); ids = arrival index, ts = id."""
        rng = np.random.default_rng(self.seed)
        total = sum(self.calls)
        if self.keys == "uniform":
            keys = rng.integers(0, self.nkeys, total).astype(np.uint64)
        else:  # "zipf:<top>": a key set spread over the slot range (and its last slot), Zipf weights over it
            ks = np.unique(np.concatenate([rng.choice(self.cap - 1, self.nkeys - 1, replace=False), [self.cap - 1]])).astype(np.uint64)
            w = 1.0 / np.arange(1, len(ks) + 1) ** float(self.keys.split(":")[1])
            keys = rng.permutation(ks)[rng.choice(len(ks), total, p=w / w.sum())]
        t = make_tuples(keys, 0, self.rec)
        out, off = [], 0
        for n in self.calls:
            out.append([(t[b:min(b + self.batch, off + n)], t["id"][b:min(b + self.batch, off + n)].copy()) for b in range(off, off + n, self.batch)])
            off += n
        return t, out

    def call_slots(self, calls):
        """Survivors' slots per call: slot = key (dense), or the order of first appearance (the key table hands slots out in turn)."""
        first = {}
        res = []
        for c in calls:
            k = np.concatenate([b[0]["key"][keep_mask(b[0])] for b in c])
            if not self.dense:
                for x in pd_unique(k):
                    first.setdefault(int(x), len(first))
                k = np.array([first[int(x)] for x in k], dtype=np.int64)
            res.append(k.astype(np.int64))
        return res


def pd_unique(a):
    _, i = np.unique(a, return_index=True)
    return a[np.sort(i)]


def _c(rec):  # record size -> geometry of a deep eager tree (log_leaves above BK_SIBL)
    return (256, 1, 1) if rec <= 32 else (24, 1, 1)


BASE_EXPECT = ("bucket_path", ("max_keys_per_bucket", 2), "multichunk_bucket", "open_pane_at_chunk", "deferred", "window_wraps_ring",
               "ring_wrapped_twice")
CASES = []
for rec in (24, 32, 48):
    nk = 64 if rec != 48 else 32  # (48-byte records: hashed 16-byte keys, all in bucket 0 and, for the thread walk, in its warp 0)
    dense = rec != 48
    CASES += [
        # multi-key buckets of several chunks, open panes across chunks, in-kernel evaluation by several lanes of a warp in the same
        # round of the thread walk, windows across the ring's end
        Case(f"r{rec}_thread_walk", rec, 48, 16, 1, 65536, nk, [24000, 24000, 24000], 4000,
             BASE_EXPECT + (("max_keys_per_bucket", nk), "inkernel_thread", "inkernel_thread_same_round"), dense=dense, seed=rec),
        # tiny-pane warp fold with in-kernel evaluation: pane 3 splits groups of 32 records; the bucket's last partial chunk takes the thread walk
        Case(f"r{rec}_tiny_pane", rec, 9, 3, 1, 65536, 64, [15000, 9000, 20000], 3000,
             ("bucket_path", "eager", "warp_fold", "warp_fold_multikey", "warp_subrange_split", "key_warp_and_thread", "inkernel_warp",
              "deferred", "window_wraps_ring", "ring_wrapped_twice"), dense=dense, seed=rec + 1),
        # eager levels above BK_SIBL through both the warp fold and (small calls) the thread walk with staged siblings
        Case(f"r{rec}_deep_eager", rec, *_c(rec), 65536, 32, [30000, 120, 25000, 100, 30000, 140, 3000], 5000 if rec <= 32 else 3000,
             ("bucket_path", "eager", "eager_above_sibl_warp", "eager_above_sibl_thread", "inkernel_warp", "deferred", "window_wraps_ring",
              "ring_wrapped_twice"), dense=dense, seed=rec + 2),
    ]
CASES += [
    # lazy levels (k_ffat_windows_lazy for the deferred groups, the leaf walk for the in-kernel ones)
    Case("r32_lazy", 32, 64, 16, 4, 65536, 64, [30000, 30000, 20000], 5000,
         ("bucket_path", "lazy", ("max_keys_per_bucket", 64), "multichunk_bucket", "inkernel_thread", "deferred_lazy", "window_wraps_ring"), seed=7),
    Case("r24_lazy_tiny_pane", 24, 10, 5, 2, 65536, 64, [20000, 12000, 20000], 4000,
         ("bucket_path", "lazy", "warp_fold", "warp_fold_multikey", "warp_subrange_split", "inkernel_warp", "deferred_lazy"), seed=8),
    # pipelined handles and the bucket-move partition
    Case("r32_thread_walk_pipelined", 32, 48, 16, 1, 65536, 64, [24000, 24000, 24000], 4000,
         ("bucket_path", "inkernel_thread", "deferred", "window_wraps_ring"), pipelined=True, seed=9),
    Case("r32_thread_walk_move", 32, 48, 16, 1, 65536, 64, [24000, 24000, 24000], 4000,
         ("bucket_path", "inkernel_thread", "deferred", "window_wraps_ring"), move=True, seed=10),
    Case("r24_tiny_pane_move", 24, 9, 3, 1, 65536, 64, [15000, 9000, 20000], 3000,
         ("bucket_path", "warp_fold", "inkernel_warp", "key_warp_and_thread"), move=True, seed=11),
    # full-sort path (light keys in k_ffat_update_lanes, Zipf heavy keys in k_ffat_update, deferred groups in k_ffat_windows)
    Case("r32_full_sort_2p17", 32, 40, 10, 2, 1 << 17, 3000, [200000, 150000, 200000], 50000,
         ("full_sort", "lanes", "update", "inkernel_lanes", "inkernel_update", "short_take_at_pane", "deferred", "window_wraps_ring"),
         keys="zipf:1.0", seed=12),
    Case("r32_full_sort_2p17_pipelined", 32, 40, 10, 2, 1 << 17, 3000, [200000, 150000, 200000], 50000,
         ("full_sort", "lanes", "update", "inkernel_lanes", "inkernel_update", "deferred"), keys="zipf:1.0", pipelined=True, seed=13),
    Case("r24_full_sort_2p20", 24, 30, 5, 3, 1 << 20, 2000, [150000, 150000], 30000,
         ("full_sort", "lanes", "update", "inkernel_lanes", "inkernel_update", "short_take_at_pane", "deferred"), keys="zipf:1.1", seed=14),
    # hashed keys at 60 000 keys (slots are handed out in a nondeterministic order: coverage only, no census)
    Case("r32_hashed_60000", 32, 4, 1, 1, 65536, 60000, [300000] * 4, 50000, (), dense=False, census=False, seed=15),
]


def _geometry(c):
    return Geometry(c.win, c.slide, c.nb, c.cap, c.rec)


def _expected(O, c, t, calls):
    """(keys, ids, ts) of the oracle's windows, sorted by (key, id), and their (h, q) by the direct fold."""
    go = O.FfatGpuOracle(c.win, c.slide, c.nb)
    exp, ets = [], []
    for call in calls:
        for tb, ts in call:
            r, rt = go.process_batch(_lift_res(tb[keep_mask(tb)]), int(ts[0]))
            exp.append(r); ets.append(rt)
    go.close()
    e, et = O.sort_results(np.concatenate(exp), np.concatenate(ets))
    surv = t[keep_mask(t)]
    order, a, b = cb_ranges(surv["key"], e["key"], e["id"], c.win, c.slide)
    h, q = hash_ranges(np_lift_h(surv, c.rec)[order], a, b, WORD[c.rec])
    return e, et, h, q, surv


def _run_cb(ops, L, prog, c, calls, out_cap=None):
    import torch
    ff = ops.FfatWindowsGPU(prog, c.win, c.slide, c.nb, max_keys=c.cap, dense_keys=c.dense, pipelined=c.pipelined)
    prm = C.c_uint64(M)
    ops.check(L.wfb_ffat_set_params(ff.h, C.byref(prm), C.sizeof(prm)), "wfb_ffat_set_params")
    got, gts = [], []
    for i, call in enumerate(calls):
        bufs = {}
        if out_cap:
            bufs = dict(out=torch.empty(out_cap * ff.res_dtype.itemsize, dtype=torch.uint8, device="cuda"),
                        out_ts=torch.empty(out_cap, dtype=torch.int64, device="cuda"))
        out, out_ts, n_out = ff.process([ops.DeviceBatch.from_host(tb, ts) for tb, ts in call], **bufs)
        torch.cuda.synchronize()
        r, rt = ff.results_to_host(out, out_ts, n_out)
        if c.pipelined and i == 0:
            assert len(r) == 0
        got.append(r); gts.append(rt)
    if c.pipelined:
        out, out_ts, n_out = ff.flush()
        torch.cuda.synchronize()
        r, rt = ff.results_to_host(out, out_ts, n_out)
        got.append(r); gts.append(rt)
    err = ff.stats()[1]
    ff.close()
    return np.concatenate(got), np.concatenate(gts), err


def _result_key(r, rec):
    return r["key"]["key"] if rec == 48 else r["key"]


def _check(got, gts, e, et, h, q, rec):
    order = np.lexsort((got["id"], _result_key(got, rec)))
    g, gt = got[order], gts[order]
    assert len(g) == len(e) > 0, (len(g), len(e))
    gk = _result_key(g, rec)
    assert np.array_equal(gk, e["key"]) and np.array_equal(g["id"], e["id"])
    assert np.array_equal(gt, et)
    if rec == 48:
        w = key16_word(e["key"])
        assert np.array_equal(g["key"]["a"], (w & np.uint64(0xffffffff)).astype(np.uint32))
        assert np.array_equal(g["key"]["b"], (w >> np.uint64(32)).astype(np.uint32))
    bad = np.flatnonzero((g["h"] != h) | (g["q"] != q))
    assert len(bad) == 0, f"{len(bad)} of {len(g)} windows differ from the direct fold, first (key, id): " \
                          f"{[(int(gk[i]), int(g['id'][i])) for i in bad[:5]]}"


@pytest.mark.parametrize("case", [c for c in CASES if c.census], ids=lambda c: c.name)
def test_case_reaches_its_regimes(case):
    """The census of every count-based case (CPU): it reaches the branches it is there for."""
    _, calls = case.stream()
    assert_regimes(census(_geometry(case), case.call_slots(calls)), case.expect)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_ordered_cb_windows_match_direct_fold(wfb, oracle, progs, monkeypatch, case):
    ops, O = wfb, oracle
    if case.move:
        monkeypatch.setenv("WFB_BUCKET_MOVE", "1")  # read when the handle is created
    t, calls = case.stream()
    g = _geometry(case)
    if case.census:
        assert_regimes(census(g, case.call_slots(calls)), case.expect)
    e, et, h, q, _ = _expected(O, case, t, calls)
    got, gts, err = _run_cb(ops, ops._lib.lib(), progs[case.rec], case, calls)
    assert err == 0
    _check(got, gts, e, et, h, q, case.rec)


# ---------------------------------------------------------------------------------------------------------------------------------
# time-based windows: the front end's pane reduce and merge, and the count-based back end on both paths
# ---------------------------------------------------------------------------------------------------------------------------------
TB_CASES = [  # name, win, slide, nb, lateness, capacity (dense keys), keys, tuples, batch, batches per call, ts step divisor, jitter
    ("bucket_back_end", 400, 100, 2, 150, 65536, 300, 120000, 2000, 6, 20, 100),
    ("full_sort_back_end", 400, 100, 2, 150, 100000, 100000, 600000, 1000, 10, 1000, 100),
]


def _tb_stream(nkeys, n, div, jitter, seed):
    rng = np.random.default_rng(seed)
    t = make_tuples(rng.integers(0, nkeys, n).astype(np.uint64), 0, 32)
    ts = (np.arange(n, dtype=np.uint64) // np.uint64(div)) + rng.integers(0, jitter, n).astype(np.uint64)
    return t, ts


@pytest.mark.gpu
@pytest.mark.parametrize("case", TB_CASES, ids=[c[0] for c in TB_CASES])
def test_ordered_tb_windows_match_direct_fold(wfb, oracle, progs, case):
    import torch
    ops, O = wfb, oracle
    name, win, slide, nb, late, cap, nkeys, n, batch, group, div, jitter = case
    t, ts = _tb_stream(nkeys, n, div, jitter, seed=len(name))
    to = O.FfatTbOracle(win, slide, late, nb)
    L = ops._lib.lib()
    ff = ops.FfatWindowsGPU(progs[32], win, slide, nb, max_keys=cap, dense_keys=True, win_type=1, lateness=late)
    prm = C.c_uint64(M)
    ops.check(L.wfb_ffat_set_params(ff.h, C.byref(prm), C.sizeof(prm)), "wfb_ffat_set_params")
    exp, ets, got, gts, batches = [], [], [], [], []
    for b in range(0, n, batch):
        tb, tsb = t[b:b + batch], ts[b:b + batch]
        k = keep_mask(tb)
        r, rt = to.process_batch(_lift_res(tb[k]), tsb[k], int(tsb[0]))
        exp.append(r); ets.append(rt)
        batches.append(ops.DeviceBatch.from_host(tb, tsb))
    assert to.ignored == 0  # nothing dropped: every item is in its windows
    for i in range(0, len(batches), group):
        out, out_ts, n_out = ff.process(batches[i:i + group])
        torch.cuda.synchronize()
        r, rt = ff.results_to_host(out, out_ts, n_out)
        got.append(r); gts.append(rt)
    assert ff.stats()[1] == 0
    e, et = O.sort_results(np.concatenate(exp), np.concatenate(ets))
    k = keep_mask(t)
    surv, sts = t[k], ts[k]
    order, a, b = tb_ranges(surv["key"], sts, e["key"], e["id"], win, slide, math.gcd(win, slide))
    h, q = hash_ranges(np_lift_h(surv, 32)[order], a, b, np.uint64)
    assert np.count_nonzero(b - a > 1) > len(e) // 2  # (most windows fold several items)
    _check(np.concatenate(got), np.concatenate(gts), e, et, h, q, 32)


# ---------------------------------------------------------------------------------------------------------------------------------
# Reduce_GPU: every key's tuples of a batch fold in arrival order (thrust::sort_by_key + reduce_by_key in the reference)
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ordered_reduce_by_key_batches(wfb, progs):
    import torch
    ops = wfb
    rng = np.random.default_rng(21)
    sizes = [5000, 0, 1, 3000, 20000, 77]
    w = 1.0 / np.arange(1, 301) ** 1.1
    eng = ops.Engine(progs[32])
    eng.set_key_bits(20)
    prm = C.c_uint64(M)
    ops.check(eng.L.wfb_engine_set_params(eng.h, C.byref(prm), C.sizeof(prm)), "wfb_engine_set_params")
    ins, outs, hosts = [], [], []
    for n in sizes:
        t = make_tuples(rng.choice(300, n, p=w / w.sum()).astype(np.uint64) * np.uint64(977), 0, 32)
        t["ivalue"] = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
        t["pad"][:, 1] = rng.integers(0, 2**63, n, dtype=np.uint64) * np.uint64(2)  # any q: the fold is over (h, q) pairs
        t["pad"][:, 2] = rng.integers(0, 2**63, n, dtype=np.uint64)
        ts = rng.permutation(n).astype(np.uint64)
        hosts.append((t, ts))
        ins.append(ops.DeviceBatch.from_host(t, ts) if n else ops.DeviceBatch(torch.empty(0, dtype=torch.uint8, device="cuda"),
                                                                            torch.empty(0, dtype=torch.int64, device="cuda"), 0, 0))
        outs.append(ops.DeviceBatch(torch.empty(max(n, 1) * 64, dtype=torch.uint8, device="cuda"),
                                    torch.empty(max(n, 1), dtype=torch.int64, device="cuda"), n, 0))
    n_out = torch.full((len(sizes),), 7, dtype=torch.int32, device="cuda")
    eng.reduce_by_key_batches(ins, outs, n_out)
    torch.cuda.synchronize()
    no = n_out.cpu().numpy()
    long_keys = 0
    for i, (t, ts) in enumerate(hosts):
        uk = np.unique(t["key"])
        assert no[i] == len(uk)
        got = ops.to_host(outs[i].tuples, TUPLE64, len(uk))
        gts = ops.ts_to_host(outs[i].ts, len(uk))
        exp = np.zeros(len(uk), dtype=TUPLE64)
        ets = np.zeros(len(uk), dtype=np.uint64)
        for j, k in enumerate(uk):
            idx = np.flatnonzero(t["key"] == k)
            long_keys += len(idx) > 48  # (segments above RB_LONG take the warp kernel)
            r = t[idx[0]].copy()
            h, q = np.array([r["ivalue"]]).view(np.uint64), np.array([r["pad"][1]], dtype=np.uint64)
            for x in idx[1:]:
                h, q = np_comb(h, q, np.array([t["ivalue"][x]]).view(np.uint64), np.array([t["pad"][x, 1]], dtype=np.uint64), np.uint64)
            r["ivalue"], r["pad"][1] = h.view(np.int64)[0], q[0]
            exp[j], ets[j] = r, ts[idx].max()
        assert got.tobytes() == exp.tobytes(), f"batch {i}"
        assert np.array_equal(gts, ets)
    assert long_keys > 0


# ---------------------------------------------------------------------------------------------------------------------------------
# the slot sort at exactly 2^24 keys: items whose key found no slot must sort behind slot 2^24 - 1, not into its run
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_full_sort_at_2p24_keys_keeps_unslotted_items_out(wfb, oracle, progs):
    ops, O = wfb, oracle
    cap, last = 1 << 24, (1 << 24) - 1
    rng = np.random.default_rng(24)
    c = Case("2p24", 32, 4, 2, 1, cap, 0, [], 0, ())
    calls = []
    nid = 0
    for n_last in (700, 200):  # slot 2^24 - 1 above light_max (k_ffat_update) in the first call, at or below it in the second
        keys = np.concatenate([np.full(n_last, last), np.full(300, cap), np.full(300, cap + 7), np.full(120, 3)]).astype(np.uint64)
        t = make_tuples(rng.permutation(keys), nid, 32)
        nid += len(t)
        calls.append([(t[b:b + 500], t["id"][b:b + 500].copy()) for b in range(0, len(t), 500)])
    surv_slots = [np.concatenate([b[0]["key"][keep_mask(b[0])] for b in call]) for call in calls]
    assert (surv_slots[0] == last).sum() > LIGHT_MAX >= (surv_slots[1] == last).sum()
    got, gts, err = _run_cb(ops, ops._lib.lib(), progs[32], c, calls, out_cap=1 << 16)
    assert err & 1  # keys 2^24 and 2^24 + 7 found no slot
    assert np.all(got["key"] < cap)
    # the reference over the windows' own keys only
    mine = [[(tb[tb["key"] < cap], ts) for tb, ts in call] for call in calls]  # (ts: the batch's watermark is ts[0])
    t_all = np.concatenate([tb for call in mine for tb, _ in call])
    e, et, h, q, _ = _expected(O, c, t_all, mine)
    assert set(np.unique(e["key"]).tolist()) == {3, last}
    _check(got, gts, e, et, h, q, 32)


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU checks
# ---------------------------------------------------------------------------------------------------------------------------------
@needs_nvcc
def test_ordered_programs_compile():
    _compile()
    assert os.path.exists(SO)


@needs_nvcc
@pytest.mark.parametrize("rec", [24, 32, 48])
def test_host_comb_matches_numpy_model(rec):
    """The programs' comb on the host == the numpy model, out aliasing an operand or not; associative on triples, not commutative,
    zero is its identity."""
    L = _ordlib()
    W = WORD[rec]
    rng = np.random.default_rng(rec)
    n = 4096
    v = [rng.integers(0, 2**63, n, dtype=np.uint64).astype(W) * W(2) + rng.integers(0, 2, n).astype(W) for _ in range(6)]
    v[1][:64] = 0; v[3][64:128] = 0  # zero lengths among the pairs

    def host(h1, q1, h2, q2, alias):
        a = [np.ascontiguousarray(x, dtype=np.uint64) for x in (h1, q1, h2, q2)]
        ho, qo = np.zeros(len(h1), np.uint64), np.zeros(len(h1), np.uint64)
        assert L.ord_comb_host(rec, M, *map(_p, a), _p(ho), _p(qo), len(h1), alias) == 0
        return ho.astype(W), qo.astype(W)
    for alias in (0, 1):
        ho, qo = host(v[0], v[1], v[2], v[3], alias)
        eh, eq = np_comb(v[0], v[1], v[2], v[3], W)
        assert np.array_equal(ho, eh) and np.array_equal(qo, eq)
    ab = np_comb(v[0], v[1], v[2], v[3], W)
    left = host(*ab, v[4], v[5], 1)
    bc = np_comb(v[2], v[3], v[4], v[5], W)
    right = host(v[0], v[1], *bc, 0)
    assert np.array_equal(left[0], right[0]) and np.array_equal(left[1], right[1])
    ba = host(v[2], v[3], v[0], v[1], 0)
    assert np.count_nonzero(ba[0] != ab[0]) > n * 0.9
    z = np.zeros(n, dtype=W)
    assert all(np.array_equal(x, y) for x, y in zip(host(z, z, v[0], v[1], 1), (v[0], v[1])))
    assert all(np.array_equal(x, y) for x, y in zip(host(v[0], v[1], z, z, 0), (v[0], v[1])))


@needs_nvcc
@pytest.mark.parametrize("rec", [24, 32, 48])
def test_host_lift_matches_numpy_model(rec):
    L = _ordlib()
    rng = np.random.default_rng(rec + 100)
    t = make_tuples(rng.integers(0, 2**64 - 2, 5000, dtype=np.uint64), int(rng.integers(0, 2**40)), rec)
    h, q, keep = np.zeros(len(t), np.uint64), np.zeros(len(t), np.uint64), np.zeros(len(t), np.uint8)
    assert L.ord_lift_host(rec, M, _p(t), len(t), _p(h), _p(q), _p(keep)) == 0
    assert np.array_equal(h.astype(WORD[rec]), np_lift_h(t, rec)) and np.all(h != 0)
    assert np.all(q == (M - 1) % (1 << _bits(WORD[rec])))
    assert np.array_equal(keep.astype(bool), keep_mask(t)) and 0 < keep.sum() < len(t)


def test_hash_ranges_equal_a_sequential_fold():
    rng = np.random.default_rng(3)
    for W in (np.uint32, np.uint64):
        h = rng.integers(0, 2**63, 300, dtype=np.uint64).astype(W)
        a = rng.integers(0, 300, 200); b = np.minimum(300, a + rng.integers(0, 40, 200))
        H, Q = hash_ranges(h, a, b, W)
        for i in range(200):
            x, y = np.zeros(1, W), np.zeros(1, W)
            for j in range(a[i], b[i]):
                x, y = np_comb(x, y, h[j:j + 1], np.array([M % (1 << _bits(W)) - 1], dtype=W), W)
            assert x[0] == H[i] and y[0] == Q[i]


@pytest.mark.parametrize("geom", [(4, 2, 1), (10, 3, 2), (48, 16, 1), (9, 3, 1), (64, 16, 4), (30, 5, 3)])
def test_direct_fold_sum_mode_matches_oracle_cb(oracle, geom):
    """The reference's window membership without a GPU: sums over the arrival ranks the direct fold uses == the oracle's isum."""
    O = oracle
    win, slide, nb = geom
    rng = np.random.default_rng(win)
    t = make_tuples(rng.integers(0, 9, 6000).astype(np.uint64), 0, 32)
    go = O.FfatGpuOracle(win, slide, nb)
    exp = [go.process_batch(_lift_res(t[b:b + 700][keep_mask(t[b:b + 700])]), b)[0] for b in range(0, len(t), 700)]
    e = O.sort_results(np.concatenate(exp))
    assert len(e) > 100
    surv = t[keep_mask(t)]
    order, a, b = cb_ranges(surv["key"], e["key"], e["id"], win, slide)
    A = np.concatenate([[0], np.cumsum(surv["id"][order].astype(np.int64))])
    assert np.array_equal(A[b] - A[a], e["isum"])


@pytest.mark.parametrize("case", TB_CASES[:1], ids=[c[0] for c in TB_CASES[:1]])
def test_direct_fold_sum_mode_matches_oracle_tb(oracle, case):
    O = oracle
    name, win, slide, nb, late, cap, nkeys, n, batch, group, div, jitter = case
    t, ts = _tb_stream(nkeys, n // 4, div, jitter, seed=3)
    to = O.FfatTbOracle(win, slide, late, nb)
    exp = []
    for b in range(0, len(t), batch):
        k = keep_mask(t[b:b + batch])
        exp.append(to.process_batch(_lift_res(t[b:b + batch][k]), ts[b:b + batch][k], int(ts[b]))[0])
    assert to.ignored == 0
    e = O.sort_results(np.concatenate(exp))
    assert len(e) > 100
    k = keep_mask(t)
    order, a, b = tb_ranges(t["key"][k], ts[k], e["key"], e["id"], win, slide, math.gcd(win, slide))
    A = np.concatenate([[0], np.cumsum(t["id"][k][order].astype(np.int64))])
    assert np.array_equal(A[b] - A[a], e["isum"])
