"""Every GPU operator across tuple, result and state sizes against a direct fold of each key's items in arrival order.

The kernels branch on the record sizes: 16-byte rotated or 8-byte tile access (TileIO), bulk or 8-byte word copies of a tile, items
per thread, cp.async granule and staged FlatFAT levels of the bucket window update, lazy or eager levels, bucket or full-sort path,
tile-pass stages. The programs of tests/cpp/record_size_programs.cu have one shape at six geometries (tuple / result / state bytes):
8/16/4, 40/40/8, 72/56/40, 128/128/128, 136/160/136 and 256/256/16. Every byte of every record depends on its inputs (map rewrites
every pad word, lift copies the tuple pad into the result pad, the window combine is an order-sensitive hash plus sums of the pad
words, the stateful functors write the state into the tuple), so a torn, short or misplaced copy shows. Outputs are compared bit for
bit, timestamps and counts exactly; the window set, ids and result timestamps come from the oracle (oracle/oracle.py), (h, q) from the
prefix hashes of tests/test_gpu_ordered_windows.py.

Batches are cut from one allocation at offsets that are 64-byte aligned or 16-byte but not 64-byte aligned, with timestamps at 0 or
8 mod 16, at sizes 0, 1, 255, 257, 4097 and 65537. A census -- a host restatement of the size conditions of wfb_kernels.cuh /
wfb_lib.cu -- asserts that the cases together reach every size branch.

CPU (-m "not gpu"): the programs compile for sm_90a, the tile pass fits the shared memory of a block at every geometry, the host
functors equal the numpy model, the model equals a plain per-key loop, and the census. GPU: everything else."""
import ctypes as C
import math
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import test_gpu_ordered_windows as ow

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "windflow_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "cpp", "record_size_programs.cu")
SO = os.path.join(ROOT, "tests", "cpp", "record_size_programs.so")
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")

GEOS = [(8, 16, 4), (40, 40, 8), (72, 56, 40), (128, 128, 128), (136, 160, 136), (256, 256, 16)]
GIDS = [f"t{t}_r{r}_s{s}" for t, r, s in GEOS]
M = ow.M
MIX0, MIX1, KMUL = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xC2B2AE3D27D4EB4F), np.uint64(0xD6E8FEB86659FD93)
TP_SMEM_MAX = 232448
SIZES = [0, 1, 255, 257, 4097, 65537]


class GeoParams(C.Structure):
    _fields_ = [("M", C.c_uint64)]


PRM = GeoParams(M)  # (wfb_engine_set_params / wfb_ffat_set_params: sizeof(params_t) bytes)


def fprm():
    """The params_t in the functor argument of a call (declared `const wfb_functors_t *`: a registered program reads its params_t there)."""
    from windflow_b200 import _lib
    return _lib.Functors.from_buffer_copy(struct.pack("<Q", M) + bytes(C.sizeof(_lib.Functors) - 8))


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
    subprocess.check_call(ow.NVCC + ["-o", SO, SRC, "-L" + os.path.join(ROOT, "windflow_b200"), "-lwfb200",
                                     "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"])


_geo = None


def geolib():
    """The test programs' shared object, loaded after libwfb200.so so that it binds the same library instance."""
    global _geo
    if _geo is None:
        _compile()
        from windflow_b200 import _lib
        _lib.lib()
        L = C.CDLL(SO)
        vp = C.c_void_p
        L.geo_register.argtypes = [C.c_int]
        L.geo_register.restype = C.c_int
        L.geo_info.argtypes = [C.c_int, vp]
        L.geo_info.restype = C.c_int
        L.geo_host.argtypes = [C.c_int, C.c_int, C.c_uint64, vp, vp, vp, C.c_uint64]
        L.geo_host.restype = C.c_int
        _geo = L
    return _geo


def info(g):
    out = np.zeros(17, dtype=np.uint32)
    assert geolib().geo_info(g, out.ctypes.data_as(C.c_void_p)) == 0
    keys = ("TB", "RB", "SB", "smem_map", "smem_filter", "smem_ingest", "smem_flatmap", "smem_lifted", "st_map", "st_filter",
            "st_ingest", "st_flatmap", "st_lifted", "bk_fits", "smem_max", "bk_smem_eager", "bk_smem_lazy")
    return dict(zip(keys, out.tolist()))


@pytest.fixture(scope="module")
def progs(wfb):
    """Program id of every geometry, with its dtypes registered in ops.RESULT_DTYPE / TUPLE_DTYPE for the module's duration."""
    L = geolib()
    ids = [L.geo_register(g) for g in range(len(GEOS))]
    assert all(i >= 6 for i in ids), ids
    for g, i in enumerate(ids):
        wfb.RESULT_DTYPE[i], wfb.TUPLE_DTYPE[i] = Geo(g).rdt, Geo(g).tdt
    yield ids
    for i in ids:
        wfb.RESULT_DTYPE.pop(i, None); wfb.TUPLE_DTYPE.pop(i, None)


# ---------------------------------------------------------------------------------------------------------------------------------
# numpy model
# ---------------------------------------------------------------------------------------------------------------------------------
class Geo:
    def __init__(self, g):
        self.g = g
        self.TB, self.RB, self.SB = GEOS[g]
        self.TP = 0 if self.TB == 8 else (self.TB - 16) // 8
        self.RP = 0 if self.RB == 16 else (self.RB - 32) // 8
        self.SP = 0 if self.SB <= 8 else (self.SB - 8) // 8
        kw = "<u4" if self.TB == 8 else "<u8"
        self.tdt = np.dtype([("key", kw), ("id", kw)] + ([("pad", "<u8", (self.TP,))] if self.TP else []))
        rw = "<u4" if self.RB == 16 else "<u8"
        self.rdt = np.dtype([("key", rw), ("id", rw), ("h", rw), ("q", rw)] + ([("pad", "<u8", (self.RP,))] if self.RP else []))
        self.WR = np.uint32 if self.RB == 16 else np.uint64
        self.WS = np.uint32 if self.SB == 4 else np.uint64
        assert self.tdt.itemsize == self.TB and self.rdt.itemsize == self.RB

    def tuples(self, keys, first_id, rng):
        t = np.zeros(len(keys), dtype=self.tdt)
        t["key"] = keys
        t["id"] = np.arange(first_id, first_id + len(keys))
        if self.TP:
            t["pad"] = rng.integers(0, 2**63, (len(keys), self.TP), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, (len(keys), self.TP)).astype(np.uint64)
        return t

    def map(self, t):
        t = t.copy()
        if self.TP:
            with np.errstate(over="ignore"):
                k = t["key"].astype(np.uint64)[:, None] * KMUL
                j = np.arange(1, self.TP + 1, dtype=np.uint64)[None, :]
                t["pad"] = (t["pad"] ^ k) + j * t["id"].astype(np.uint64)[:, None]
        return t

    @staticmethod
    def keep(t):
        return t["id"] % 7 != 3

    @staticmethod
    def mix(t):
        with np.errstate(over="ignore"):
            x = ((t["id"].astype(np.uint64) + np.uint64(1)) * MIX0) ^ (t["key"].astype(np.uint64) * MIX1)
            x ^= x >> np.uint64(29)
            return x | np.uint64(1)

    def lift(self, t):
        r = np.zeros(len(t), dtype=self.rdt)
        r["key"] = t["key"]
        r["h"] = self.mix(t).astype(self.WR)
        r["q"] = self.WR((M - 1) % (1 << (8 * np.dtype(self.WR).itemsize)))
        if self.RP:
            with np.errstate(over="ignore"):
                r["pad"] = t["pad"][:, np.arange(self.RP) % self.TP] + np.arange(self.RP, dtype=np.uint64)[None, :]
        return r

    def comb(self, a, b):
        o = a.copy()
        o["h"], o["q"] = ow.np_comb(a["h"], a["q"], b["h"], b["q"], self.WR)
        if self.RP:
            with np.errstate(over="ignore"):
                o["pad"] = a["pad"] + b["pad"]
        return o

    def reduce_fold(self, t):
        """Reduce functor folded over t in order, starting from t[0] (plain Python integers)."""
        r = t[0].copy()
        if self.TB == 8:
            h, q = int(r["id"]) & 0xffff, int(r["id"]) >> 16
            for x in t["id"][1:].tolist():
                h, q = (h * ((x >> 16) + 1) + (x & 0xffff)) & 0xffff, ((q + 1) * ((x >> 16) + 1) - 1) & 0xffff
            r["id"] = h | (q << 16)
            return r
        m64 = (1 << 64) - 1
        h, q = int(r["pad"][0]), int(r["pad"][1])
        for h2, q2 in t["pad"][1:, :2].tolist():
            h, q = (h * (q2 + 1) + h2) & m64, ((q + 1) * (q2 + 1) - 1) & m64
        r["pad"][0], r["pad"][1] = h, q
        if self.TP > 2:
            with np.errstate(over="ignore"):
                r["pad"][2:] = t["pad"][:, 2:].sum(axis=0, dtype=np.uint64)
        return r

    def reduce_pair(self, a, b):
        return self.reduce_fold(np.concatenate([a[None], b[None]]))

    def stateful(self, t):
        """Keyed-stateful map over the sequence t (states from zero): (tuples out, filter flags). Vectorised with per-key prefix
        hashes / sums."""
        n = len(t)
        order = np.argsort(t["key"], kind="stable")
        sk = t["key"][order]
        start = np.zeros(n, dtype=np.int64)
        if n:
            first = np.concatenate([[True], sk[1:] != sk[:-1]])
            start = np.maximum.accumulate(np.where(first, np.arange(n), 0))
        pos = np.arange(n)
        h = np.zeros(n, dtype=self.WS)
        h[order] = ow.hash_ranges(self.mix(t[order]).astype(self.WS), start, pos + 1, self.WS)[0]
        out = t.copy()
        if self.TB == 8:
            out["id"] = h.astype(np.uint32)
        else:
            hh = h.astype(np.uint64)
            with np.errstate(over="ignore"):
                out["pad"][:, 0] = hh
                for j in range(1, self.TP):
                    out["pad"][:, j] += hh * np.uint64(j)
                ids, ks = t["id"][order].astype(np.uint64), t["key"][order].astype(np.uint64)
                for i in range(self.SP):
                    c = np.cumsum(ids * np.uint64(2 * i + 1) + ks, dtype=np.uint64)
                    s = np.zeros(n, dtype=np.uint64)
                    s[order] = c - np.concatenate([[np.uint64(0)], c])[start]
                    out["pad"][:, 1 + i % (self.TP - 1)] ^= s
        keep = ((h.astype(np.uint64) >> np.uint64(13)) & np.uint64(3)) != 0
        return out, keep

    def stateful_loop(self, t):
        """The same, item after item with a per-key state (plain Python integers)."""
        bits = 32 if self.SB == 4 else 64
        mask = (1 << bits) - 1
        m64 = (1 << 64) - 1
        st = {}
        out, keep = t.copy(), np.zeros(len(t), dtype=bool)
        xs = self.mix(t).tolist()
        for i in range(len(t)):
            k, idv = int(t["key"][i]), int(t["id"][i])
            h, pad = st.get(k, (0, [0] * self.SP))
            h = (h * (M & mask) + (xs[i] & mask)) & mask
            pad = [(p + idv * (2 * j + 1) + k) & m64 for j, p in enumerate(pad)]
            st[k] = (h, pad)
            if self.TB == 8:
                out["id"][i] = h
            else:
                p = [int(v) for v in t["pad"][i]]
                p[0] = h
                for j in range(1, self.TP):
                    p[j] = (p[j] + h * j) & m64
                for j, v in enumerate(pad):
                    p[1 + j % (self.TP - 1)] ^= v
                out["pad"][i] = p
            keep[i] = ((h >> 13) & 3) != 0
        return out, keep

    def flatmap(self, t, ts):
        u = self.map(t)
        k = self.keep(u)
        u, uts = u[k], ts[k]
        c = (u["id"] % 3).astype(np.int64)
        idx = np.repeat(np.arange(len(u)), c)
        j = np.arange(int(c.sum())) - np.repeat(np.cumsum(c) - c, c)
        r = self.lift(u[idx])
        r["id"] = j
        return r, uts[idx]


# ---------------------------------------------------------------------------------------------------------------------------------
# census: the size branches of the kernels (host restatement of wfb_kernels.cuh / wfb_lib.cu)
# ---------------------------------------------------------------------------------------------------------------------------------
def size_tags(TB, RB):
    tags = set()
    v16 = TB % 16 == 0 and TB // 16 in (1, 2, 4, 8)
    tags.add(f"tileio_v16_c{TB // 16}" if v16 else "tileio_8b")                          # TileIO<T>
    tags.add("rec_uint4" if TB % 16 == 0 else "rec_uint2")                                # ld_rec / st_rec of tuples
    IT = min(8, max(1, 16384 // (128 * RB)))                                              # bk_items_per_thread
    tags.add(f"IT{IT}")
    tags.add(f"CPB{16 if RB % 16 == 0 else 8}")
    tags.add(f"BK_SIBL{8 if RB <= 32 else (4 if RB <= 48 else (2 if RB <= 128 else 1))}")
    return tags


def tile_tags(TB, addr, n, ts_addr):
    """Tile-copy branches of the tile pass over one batch at device offset addr (timestamps at ts_addr, None: none)."""
    tags = set()
    for first in range(0, n, 256):
        cnt = min(256, n - first)
        src = addr + first * TB
        tags.add("tile_bulk" if (src | cnt * TB) % 16 == 0 else "tile_fallback")
        if ts_addr is not None:
            tags.add("ts_smem" if (ts_addr + 8 * first) % 16 == 0 and (cnt * 8) % 16 == 0 else "ts_words")
    return tags


def window_tags(RB, win, slide, nb, cap, has_buckets):
    g = ow.Geometry(win, slide, nb, cap, RB)
    buckets = g.buckets and has_buckets
    fits = buckets and 2 * g.n * RB <= (32 << 10)
    lazy = fits and g.n <= 2 * max(1, g.logn) * g.sp * nb
    return {"bucket_path" if buckets else "full_sort", ("lazy" if lazy else "eager")}


# ---------------------------------------------------------------------------------------------------------------------------------
# batches in one allocation
# ---------------------------------------------------------------------------------------------------------------------------------
def layout(sizes, TB, align):
    """Byte offsets of the batches in one allocation: 64-byte aligned (align 64) or 16 mod 64 (align 16); timestamps at 0 mod 16
    (align 64) or 8 mod 16 (align 16), as element offsets of an int64 buffer."""
    offs, tso, o, to = [], [], 0, 0
    for n in sizes:
        o = (o + 63) // 64 * 64 + (16 if align == 16 else 0)
        to = (to + 1) // 2 * 2 + (1 if align == 16 else 0)
        offs.append(o); tso.append(to)
        o += n * TB + 8; to += n + 1
    return offs, tso, o + 64, to + 2


def upload(ops, arrs, tss, TB, align, fill=0xAB):
    """DeviceBatch views into one tuple and one timestamp allocation (guard bytes around every batch)."""
    import torch
    offs, tso, nb, nt = layout([len(a) for a in arrs], TB, align)
    buf = np.full(nb, fill, dtype=np.uint8)
    tsb = np.full(nt, -1, dtype=np.int64)
    for a, ts, o, to in zip(arrs, tss, offs, tso):
        buf[o:o + len(a) * TB] = np.frombuffer(np.ascontiguousarray(a).tobytes(), dtype=np.uint8)
        tsb[to:to + len(a)] = np.asarray(ts, dtype=np.uint64).view(np.int64)
    dbuf, dts = torch.from_numpy(buf).cuda(), torch.from_numpy(tsb).cuda()
    bs = [ops.DeviceBatch(dbuf[o:o + max(1, len(a)) * TB], dts[to:to + max(1, len(a))], len(a), int(ts[0]) if len(a) else 0)
          for a, ts, o, to in zip(arrs, tss, offs, tso)]
    return bs, dbuf, dts, offs, tso


def empty_like_layout(ops, sizes, TB, align, fill=0xCD):
    import torch
    offs, tso, nb, nt = layout(sizes, TB, align)
    dbuf = torch.full((nb,), fill, dtype=torch.uint8, device="cuda")
    dts = torch.full((nt,), -1, dtype=torch.int64, device="cuda")
    bs = [ops.DeviceBatch(dbuf[o:o + max(1, n) * TB], dts[to:to + max(1, n)], n, 0) for n, o, to in zip(sizes, offs, tso)]
    return bs, dbuf, dts, offs, tso


def batches_of(geo, sizes, nkeys, seed, first_id=0):
    rng = np.random.default_rng(seed)
    arrs, tss, nid = [], [], first_id
    for n in sizes:
        arrs.append(geo.tuples(rng.integers(0, nkeys, n).astype(np.uint64), nid, rng))
        tss.append(rng.integers(0, 1 << 40, n, dtype=np.uint64))
        nid += n
    return arrs, tss


def host_bytes(dbuf, off, n, TB):
    return dbuf[off:off + n * TB].cpu().numpy().tobytes()


def guards_intact(dbuf, offs, sizes, TB, fill):
    raw = dbuf.cpu().numpy()
    mask = np.ones(len(raw), dtype=bool)
    for o, n in zip(offs, sizes):
        mask[o:o + n * TB] = False
    return bool((raw[mask] == fill).all())


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU checks
# ---------------------------------------------------------------------------------------------------------------------------------
@needs_nvcc
def test_programs_compile():
    _compile()
    assert os.path.exists(SO)


@needs_nvcc
@pytest.mark.parametrize("g", range(len(GEOS)), ids=GIDS)
def test_tile_pass_fits_shared_memory(g):
    """Every mode of the tile pass (and the lifted program's ingest) fits the opt-in shared memory of a block; large records keep
    fewer stages; the bucket window update exists up to 160-byte results."""
    d = info(g)
    assert d["smem_max"] == TP_SMEM_MAX
    for m in ("map", "filter", "ingest", "flatmap", "lifted"):
        assert d[f"smem_{m}"] <= TP_SMEM_MAX, (m, d)
        assert d[f"st_{m}"] in (2, 3, 4)
    TB, RB = GEOS[g][:2]
    if TB <= 128 and RB <= 128:
        assert all(d[f"st_{m}"] == 4 for m in ("map", "filter", "ingest", "flatmap", "lifted")), d
    if TB == 256:
        assert d["st_map"] == d["st_filter"] == d["st_ingest"] == 3, d
    assert d["bk_fits"] == (1 if RB <= 160 else 0)
    assert (d["bk_smem_eager"] <= 48 << 10) == (RB <= 160)


@needs_nvcc
@pytest.mark.parametrize("g", range(len(GEOS)), ids=GIDS)
def test_host_functors_match_numpy_model(g):
    L, geo = geolib(), Geo(g)
    rng = np.random.default_rng(g)
    n = 3000
    t = geo.tuples(rng.integers(0, 50, n).astype(np.uint64), int(rng.integers(0, 2**30)), rng)

    def host(op, a, b=None, out=None, nn=n):
        p = [x.ctypes.data_as(C.c_void_p) if x is not None else None for x in (a, b, out)]
        assert L.geo_host(g, op, M, p[0], p[1], p[2], nn) == 0
    m = t.copy(); host(0, m)
    assert m.tobytes() == geo.map(t).tobytes()
    keep = np.zeros(n, np.uint8); host(1, t.copy(), None, keep)
    assert np.array_equal(keep.astype(bool), geo.keep(t)) and 0 < keep.sum() < n
    r = np.zeros(n, geo.rdt); host(2, t.copy(), None, r)
    assert r.tobytes() == geo.lift(t).tobytes()
    a, b = geo.lift(t), geo.lift(t[::-1].copy())
    a["q"] = rng.integers(0, 2**31, n).astype(geo.WR)
    o = a.copy(); o["h"], o["q"] = 0, 0; host(3, a.copy(), b, o)  # (comb writes h, q and pad: key and id stay)
    assert o.tobytes() == geo.comb(a, b).tobytes()
    al = a.copy(); host(4, al, b)
    assert al.tobytes() == geo.comb(a, b).tobytes()
    assert geo.comb(a, b).tobytes() != geo.comb(b, a).tobytes()
    z = a.copy(); z["h"], z["q"] = 0, 0  # (a zero payload with a's key and id)
    if geo.RP:
        z["pad"] = 0
    assert geo.comb(z, a).tobytes() == geo.comb(a, z).tobytes() == a.tobytes()
    u = t[::-1].copy()
    rr = np.zeros(n, geo.tdt); host(5, t.copy(), u, rr)
    assert rr.tobytes() == np.concatenate([geo.reduce_pair(t[i], u[i])[None] for i in range(n)]).tobytes()
    ms = t.copy(); host(6, ms)
    exp, ek = geo.stateful(t)
    assert ms.tobytes() == exp.tobytes()
    fs, fk = t.copy(), np.zeros(n, np.uint8); host(7, fs, None, fk)
    assert fs.tobytes() == exp.tobytes() and np.array_equal(fk.astype(bool), ek) and 0 < fk.sum() < n


@pytest.mark.parametrize("g", range(len(GEOS)), ids=GIDS)
def test_stateful_model_equals_per_key_loop(g):
    geo = Geo(g)
    rng = np.random.default_rng(g + 50)
    t = geo.tuples(rng.integers(0, 40, 2000).astype(np.uint64), 7, rng)
    a, ak = geo.stateful(t)
    b, bk = geo.stateful_loop(t)
    assert a.tobytes() == b.tobytes() and np.array_equal(ak, bk)


@pytest.mark.parametrize("g", range(len(GEOS)), ids=GIDS)
def test_window_pad_model_equals_sequential_fold(g):
    """The windows' expected records (prefix hashes and prefix sums over ranges) equal a fold with the model's comb."""
    geo = Geo(g)
    rng = np.random.default_rng(g + 70)
    t = geo.tuples(rng.integers(0, 1, 300).astype(np.uint64), 0, rng)
    lifted = geo.lift(geo.map(t))
    a = rng.integers(0, 300, 60); b = np.minimum(300, a + rng.integers(0, 30, 60))
    exp = expected_records(geo, lifted, np.arange(300), a, b, np.zeros(60, np.uint64), np.arange(60))
    for i in range(60):
        r = np.zeros(1, geo.rdt)
        for j in range(a[i], b[i]):
            r = geo.comb(r, lifted[j:j + 1])
        r["id"] = i
        assert r.tobytes() == exp[i:i + 1].tobytes()


# ---------------------------------------------------------------------------------------------------------------------------------
# window cases
# ---------------------------------------------------------------------------------------------------------------------------------
class WCase:
    def __init__(self, name, win, slide, nb, cap, nkeys, calls, batch, dense=True, pipelined=False, keys="uniform", seed=1):
        self.name, self.win, self.slide, self.nb, self.cap, self.nkeys = name, win, slide, nb, cap, nkeys
        self.calls, self.batch, self.dense, self.pipelined, self.keys, self.seed = calls, batch, dense, pipelined, keys, seed


WCASES = [
    WCase("small_eager", 48, 16, 1, 65536, 64, [12000, 257, 12000], 4000, seed=1),
    WCase("small_lazy", 64, 16, 4, 65536, 64, [15000, 15000], 5000, seed=2),
    WCase("bench_geometry", 4096, 64, 65, 65536, 4, [20000, 25000], 5000, seed=3),  # lazy up to 64-byte results, eager above
    WCase("full_sort", 40, 10, 2, 1 << 17, 2000, [40000, 30000], 10000, keys="zipf", seed=4),
    WCase("small_eager_pipelined", 48, 16, 1, 65536, 64, [12000, 12000, 4097], 4000, pipelined=True, seed=5),
]


def expected_records(geo, lifted, order, a, b, keys, ids):
    """Window records over the lifted items (in range order `order`): ranges [a, b) -> (h, q) by prefix hashes, pad by prefix sums."""
    e = np.zeros(len(a), dtype=geo.rdt)
    e["key"], e["id"] = keys, ids
    L = lifted[order]
    e["h"], e["q"] = ow.hash_ranges(L["h"].astype(geo.WR), a, b, geo.WR)
    if geo.RP:
        with np.errstate(over="ignore"):
            P = np.zeros((len(L) + 1, geo.RP), dtype=np.uint64)
            P[1:] = np.cumsum(L["pad"], axis=0, dtype=np.uint64)
            e["pad"] = P[b] - P[a]
    return e


def _wstream(geo, c):
    rng = np.random.default_rng(c.seed)
    total = sum(c.calls)
    if c.keys == "uniform":
        keys = rng.integers(0, c.nkeys, total).astype(np.uint64)
    else:
        ks = rng.choice(c.cap, c.nkeys, replace=False).astype(np.uint64)
        w = 1.0 / np.arange(1, len(ks) + 1) ** 1.0
        keys = ks[rng.choice(len(ks), total, p=w / w.sum())]
    t = geo.tuples(keys, 0, rng)
    calls, off = [], 0
    for n in c.calls:
        calls.append([(t[s:min(s + c.batch, off + n)], t["id"][s:min(s + c.batch, off + n)].astype(np.uint64)) for s in range(off, off + n, c.batch)])
        off += n
    return t, calls


def _check_windows(geo, got, gts, e, et):
    order = np.lexsort((got["id"], got["key"]))
    g, gt = got[order], gts[order]
    eo = np.lexsort((e["id"], e["key"]))
    e, et = e[eo], et[eo]
    assert len(g) == len(e) > 0, (len(g), len(e))
    assert np.array_equal(gt, et)
    gb, eb = g.view(np.uint8).reshape(len(g), -1), e.view(np.uint8).reshape(len(e), -1)
    bad = np.flatnonzero((gb != eb).any(axis=1))
    assert len(bad) == 0, f"{len(bad)} of {len(g)} windows differ from the direct fold, first (key, id): " \
                          f"{[(int(g['key'][i]), int(g['id'][i])) for i in bad[:5]]}"


def _expected_cb(O, geo, c, t, calls):
    go = O.FfatGpuOracle(c.win, c.slide, c.nb)
    exp, ets = [], []
    for call in calls:
        for tb, ts in call:
            r, rt = go.process_batch(ow._lift_res(tb[geo.keep(tb)]), int(ts[0]))
            exp.append(r); ets.append(rt)
    go.close()
    e, et = O.sort_results(np.concatenate(exp), np.concatenate(ets))
    surv = geo.map(t)[geo.keep(t)]
    order, a, b = ow.cb_ranges(surv["key"].astype(np.uint64), e["key"], e["id"], c.win, c.slide)
    return expected_records(geo, geo.lift(surv), order, a, b, e["key"], e["id"]), et


@pytest.mark.parametrize("c", WCASES, ids=lambda c: c.name)
def test_window_case_reaches_its_path(c):
    """(CPU) the path every window case takes at every geometry: the bench geometry flips from lazy to eager levels above
    64-byte results; results above 160 bytes take the full-sort path."""
    for TB, RB, SB in GEOS:
        tags = window_tags(RB, c.win, c.slide, c.nb, c.cap, RB <= 160)
        if c.name == "full_sort" or RB > 160:
            assert tags == {"full_sort", "eager"}, (RB, tags)
        elif c.name == "small_lazy":
            assert tags == {"bucket_path", "lazy"}
        elif c.name == "bench_geometry":
            assert tags == {"bucket_path", "lazy" if RB <= 64 else "eager"}, (RB, tags)
        else:
            assert tags == {"bucket_path", "eager"}


@pytest.mark.gpu
@pytest.mark.parametrize("c", WCASES, ids=lambda c: c.name)
@pytest.mark.parametrize("g", range(len(GEOS)), ids=GIDS)
def test_cb_windows_match_direct_fold(wfb, oracle, progs, g, c):
    import torch
    ops, geo = wfb, Geo(g)
    t, calls = _wstream(geo, c)
    e, et = _expected_cb(oracle, geo, c, t, calls)
    ff = ops.FfatWindowsGPU(progs[g], c.win, c.slide, c.nb, max_keys=c.cap, dense_keys=c.dense, pipelined=c.pipelined)
    ops.check(ff.L.wfb_ffat_set_params(ff.h, C.byref(PRM), C.sizeof(PRM)), "wfb_ffat_set_params")
    got, gts = [], []
    for i, call in enumerate(calls):
        bs = upload(ops, [x for x, _ in call], [y for _, y in call], geo.TB, 16 if i % 2 else 64)[0]
        out, out_ts, n_out = ff.process(bs)
        torch.cuda.synchronize()
        r, rt = ff.results_to_host(out, out_ts, n_out)
        got.append(r); gts.append(rt)
    if c.pipelined:
        out, out_ts, n_out = ff.flush()
        torch.cuda.synchronize()
        r, rt = ff.results_to_host(out, out_ts, n_out)
        got.append(r); gts.append(rt)
    assert ff.stats()[1] == 0
    ff.close()
    _check_windows(geo, np.concatenate(got), np.concatenate(gts), e, et)


@pytest.mark.gpu
@pytest.mark.parametrize("g", range(len(GEOS)), ids=GIDS)
def test_tb_windows_match_direct_fold(wfb, oracle, progs, g):
    import torch
    ops, O, geo = wfb, oracle, Geo(g)
    win, slide, nb, late, cap, nkeys, n, batch, group, div, jitter = 400, 100, 2, 150, 65536, 300, 60000, 2000, 6, 20, 100
    rng = np.random.default_rng(g + 90)
    t = geo.tuples(rng.integers(0, nkeys, n).astype(np.uint64), 0, rng)
    ts = (np.arange(n, dtype=np.uint64) // np.uint64(div)) + rng.integers(0, jitter, n).astype(np.uint64)
    to = O.FfatTbOracle(win, slide, late, nb)
    ff = ops.FfatWindowsGPU(progs[g], win, slide, nb, max_keys=cap, dense_keys=True, win_type=1, lateness=late)
    ops.check(ff.L.wfb_ffat_set_params(ff.h, C.byref(PRM), C.sizeof(PRM)), "wfb_ffat_set_params")
    exp, ets, got, gts, arrs, tss = [], [], [], [], [], []
    for b in range(0, n, batch):
        tb, tsb = t[b:b + batch], ts[b:b + batch]
        k = geo.keep(tb)
        r, rt = to.process_batch(ow._lift_res(tb[k]), tsb[k], int(tsb[0]))
        exp.append(r); ets.append(rt)
        arrs.append(tb); tss.append(tsb)
    assert to.ignored == 0
    for i in range(0, len(arrs), group):
        bs = upload(ops, arrs[i:i + group], tss[i:i + group], geo.TB, 16 if (i // group) % 2 else 64)[0]
        out, out_ts, n_out = ff.process(bs)
        torch.cuda.synchronize()
        r, rt = ff.results_to_host(out, out_ts, n_out)
        got.append(r); gts.append(rt)
    assert ff.stats()[1] == 0
    ff.close()
    e, et = O.sort_results(np.concatenate(exp), np.concatenate(ets))
    k = geo.keep(t)
    surv, sts = geo.map(t)[k], ts[k]
    order, a, b = ow.tb_ranges(surv["key"].astype(np.uint64), sts, e["key"], e["id"], win, slide, math.gcd(win, slide))
    ee = expected_records(geo, geo.lift(surv), order, a, b, e["key"], e["id"])
    assert np.count_nonzero(b - a > 1) > len(e) // 2
    _check_windows(geo, np.concatenate(got), np.concatenate(gts), ee, et)


# ---------------------------------------------------------------------------------------------------------------------------------
# Map / Filter / FlatMap
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("align", [64, 16])
@pytest.mark.parametrize("g", range(len(GEOS)), ids=GIDS)
def test_map(wfb, progs, g, align):
    import torch
    ops, geo = wfb, Geo(g)
    arrs, tss = batches_of(geo, SIZES, 1000, seed=g)
    bs, dbuf, _, offs, _ = upload(ops, arrs, tss, geo.TB, align)
    eng = ops.Engine(progs[g])
    for b in bs:
        eng.map(b, fprm())
    torch.cuda.synchronize()
    for a, o in zip(arrs, offs):
        assert host_bytes(dbuf, o, len(a), geo.TB) == geo.map(a).tobytes(), len(a)
    assert guards_intact(dbuf, offs, SIZES, geo.TB, 0xAB)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("inplace", [False, True], ids=["out_of_place", "in_place"])
@pytest.mark.parametrize("align", [64, 16])
@pytest.mark.parametrize("g", range(len(GEOS)), ids=GIDS)
def test_map_filter_batches(wfb, progs, g, align, inplace):
    import torch
    ops, geo = wfb, Geo(g)
    arrs, tss = batches_of(geo, SIZES, 1000, seed=g + 10)
    bs, dbuf, dts, offs, tso = upload(ops, arrs, tss, geo.TB, align)
    if inplace:
        outs, obuf, ots, ooffs, otso = bs, dbuf, dts, offs, tso
    else:
        outs, obuf, ots, ooffs, otso = empty_like_layout(ops, SIZES, geo.TB, 80 - align)  # (the other alignment)
    n_out = torch.full((len(bs),), 7, dtype=torch.int32, device="cuda")
    eng = ops.Engine(progs[g])
    eng.map_filter_batches(bs, fprm(), outs, n_out)
    torch.cuda.synchronize()
    no = n_out.cpu().numpy()
    tsh = ots.cpu().numpy().view(np.uint64)
    for i, (a, ts) in enumerate(zip(arrs, tss)):
        u = geo.map(a)
        k = geo.keep(u)
        assert no[i] == k.sum()
        assert host_bytes(obuf, ooffs[i], int(no[i]), geo.TB) == u[k].tobytes(), (i, len(a))
        assert np.array_equal(tsh[otso[i]:otso[i] + no[i]], ts[k])
    if not inplace:
        assert guards_intact(obuf, ooffs, no.tolist(), geo.TB, 0xCD)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("g", range(len(GEOS)), ids=GIDS)
def test_flatmap_batches(wfb, progs, g):
    import torch
    ops, geo = wfb, Geo(g)
    sizes = [1, 255, 257, 4097, 0, 20000]
    arrs, tss = batches_of(geo, sizes, 1000, seed=g + 20)
    bs = upload(ops, arrs, tss, geo.TB, 16)[0]
    outs, obuf, ots, ooffs, otso = empty_like_layout(ops, [2 * n for n in sizes], geo.RB, 64)
    n_out = torch.full((len(bs) + 1,), 7, dtype=torch.int32, device="cuda")
    eng = ops.Engine(progs[g])
    eng.flatmap_batches(bs, fprm(), outs, n_out, 2)
    torch.cuda.synchronize()
    no = n_out.cpu().numpy()
    tsh = ots.cpu().numpy().view(np.uint64)
    assert no[-1] == 0
    for i, (a, ts) in enumerate(zip(arrs, tss)):
        r, rts = geo.flatmap(a, ts)
        assert no[i] == len(r)
        assert host_bytes(obuf, ooffs[i], len(r), geo.RB) == r.tobytes(), i
        assert np.array_equal(tsh[otso[i]:otso[i] + len(r)], rts)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# keyed-stateful Map / Filter
# ---------------------------------------------------------------------------------------------------------------------------------
STATEFUL = [("buckets", 65536, 3000, [[4097, 0, 255, 1, 20000], [257, 30000]]),
            ("sort", 1 << 17, 100000, [[65537, 1, 255], [257, 120000]])]


@pytest.mark.gpu
@pytest.mark.parametrize("case", STATEFUL, ids=[s[0] for s in STATEFUL])
@pytest.mark.parametrize("g", range(len(GEOS)), ids=GIDS)
def test_keyed_stateful(wfb, progs, g, case):
    import torch
    ops, geo = wfb, Geo(g)
    name, cap, nkeys, calls = case
    rng = np.random.default_rng(g + 30)
    keyset = rng.choice(1 << 31, nkeys, replace=False).astype(np.uint64)
    total = sum(sum(c) for c in calls)
    t = geo.tuples(keyset[rng.integers(0, nkeys, total)], 0, rng)
    ts = rng.integers(0, 1 << 40, total, dtype=np.uint64)
    exp, ek = geo.stateful(t)
    assert len(np.unique(t["key"])) > (65536 if name == "sort" else 1000)
    km, kf = ops.KeyedState(progs[g], cap), ops.KeyedState(progs[g], cap)
    off = 0
    for ci, sizes in enumerate(calls):
        arrs = [t[off + sum(sizes[:i]):off + sum(sizes[:i + 1])] for i in range(len(sizes))]
        tss = [ts[off + sum(sizes[:i]):off + sum(sizes[:i + 1])] for i in range(len(sizes))]
        align = 16 if ci % 2 else 64
        bs, dbuf, _, offs, _ = upload(ops, arrs, tss, geo.TB, align)
        km.map(bs, fprm())
        fb = upload(ops, arrs, tss, geo.TB, align)[0]
        outs, obuf, ots, ooffs, otso = empty_like_layout(ops, sizes, geo.TB, 80 - align)
        n_out = torch.full((len(fb),), 7, dtype=torch.int32, device="cuda")
        kf.filter(fb, fprm(), outs, n_out)
        torch.cuda.synchronize()
        no = n_out.cpu().numpy()
        tsh = ots.cpu().numpy().view(np.uint64)
        p = off
        for i, (a, tb) in enumerate(zip(arrs, tss)):
            n = len(a)
            assert host_bytes(dbuf, offs[i], n, geo.TB) == exp[p:p + n].tobytes(), (ci, i, n)
            k = ek[p:p + n]
            assert no[i] == k.sum(), (ci, i)
            assert host_bytes(obuf, ooffs[i], int(no[i]), geo.TB) == exp[p:p + n][k].tobytes(), (ci, i, n)
            assert np.array_equal(tsh[otso[i]:otso[i] + no[i]], tb[k])
            p += n
        assert guards_intact(dbuf, offs, sizes, geo.TB, 0xAB)
        off += sum(sizes)
    km.close(); kf.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# Reduce_GPU
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("g", range(len(GEOS)), ids=GIDS)
def test_reduce_by_key_batches(wfb, progs, g):
    import torch
    ops, geo = wfb, Geo(g)
    rng = np.random.default_rng(g + 40)
    w = 1.0 / np.arange(1, 301) ** 1.1
    arrs, tss = [], []
    for n in SIZES:
        a = geo.tuples((rng.choice(300, n, p=w / w.sum()) * 977).astype(np.uint64), 0, rng)
        if geo.TB == 8:
            a["id"] = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
        arrs.append(a); tss.append(rng.permutation(n).astype(np.uint64))
    bs = upload(ops, arrs, tss, geo.TB, 16)[0]
    outs, obuf, ots, ooffs, otso = empty_like_layout(ops, SIZES, geo.TB, 64)
    n_out = torch.full((len(bs),), 7, dtype=torch.int32, device="cuda")
    eng = ops.Engine(progs[g])
    eng.set_key_bits(20)
    ops.check(eng.L.wfb_engine_set_params(eng.h, C.byref(PRM), C.sizeof(PRM)), "wfb_engine_set_params")
    eng.reduce_by_key_batches(bs, outs, n_out)
    torch.cuda.synchronize()
    no = n_out.cpu().numpy()
    tsh = ots.cpu().numpy().view(np.uint64)
    for i, (a, ts) in enumerate(zip(arrs, tss)):
        uk = np.unique(a["key"])
        assert no[i] == len(uk)
        order = np.argsort(a["key"], kind="stable")
        starts = np.searchsorted(a["key"][order], uk)
        ends = np.append(starts[1:], len(a))
        exp = np.concatenate([geo.reduce_fold(a[order[s:e]])[None] for s, e in zip(starts, ends)]) if len(uk) else a[:0]
        assert host_bytes(obuf, ooffs[i], len(uk), geo.TB) == exp.tobytes(), i
        assert np.array_equal(tsh[otso[i]:otso[i] + len(uk)], np.array([ts[order[s:e]].max() for s, e in zip(starts, ends)], dtype=np.uint64))
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("g", range(len(GEOS)), ids=GIDS)
def test_reduce_all(wfb, progs, g):
    ops, geo = wfb, Geo(g)
    arrs, tss = batches_of(geo, SIZES, 50, seed=g + 60)
    bs = upload(ops, arrs, tss, geo.TB, 16)[0]
    eng = ops.Engine(progs[g])
    ops.check(eng.L.wfb_engine_set_params(eng.h, C.byref(PRM), C.sizeof(PRM)), "wfb_engine_set_params")
    for a, ts, b in zip(arrs, tss, bs):
        out_t, out_ts = eng.reduce_all(b)
        exp = geo.reduce_fold(np.concatenate([np.zeros(1, geo.tdt), a]))  # (the fold starts from a zero tuple)
        assert out_t.cpu().numpy().tobytes() == exp.tobytes(), len(a)
        assert int(out_ts.cpu().numpy().view(np.uint64)[0]) == (int(ts.max()) if len(a) else 0)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# census: the cases above reach every size branch
# ---------------------------------------------------------------------------------------------------------------------------------
def census_all():
    tags = set()
    for TB, RB, SB in GEOS:
        tags |= size_tags(TB, RB)
        for align in (64, 16):
            offs, tso, _, _ = layout(SIZES, TB, align)
            for o, to, n in zip(offs, tso, SIZES):
                tags |= tile_tags(TB, o, n, 8 * to)
        for c in WCASES:
            tags |= window_tags(RB, c.win, c.slide, c.nb, c.cap, RB <= 160)
    return tags


def test_census_reaches_every_size_branch():
    tags = census_all()
    want = {"tileio_8b", "tileio_v16_c8", "rec_uint4", "rec_uint2", "IT8", "IT3", "IT2", "IT1", "CPB16", "CPB8", "BK_SIBL8", "BK_SIBL4",
            "BK_SIBL2", "BK_SIBL1", "tile_bulk", "tile_fallback", "ts_smem", "ts_words", "bucket_path", "full_sort", "lazy", "eager"}
    assert want <= tags, f"not reached: {sorted(want - tags)}"
