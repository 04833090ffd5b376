"""The code paths of blocks above 1 GiB, run on small blocks and checked against the reference.

In production only blocks above 1 GiB reach them: an in-place bsc_compress with the BWT (compress_large: a context of its own, one arena,
LZP on the host, the caller's buffer written only on success), bsc_decompress of a BWT block on a context of its own, and bsc_decompress
of an ST3..ST8 block through the lean layout of the inverse ST (decompress_large_st: st_heads_lean, st_serial_lean and st_place_lean write
in place over arrays that other steps still read).  BSCB200_LARGE_N=<bytes> lowers the threshold for one process, so the same paths meet
every input class the pooled path is checked on.  Each threshold runs in a child process of its own (tests/gpu_child.py):

  routed   BSCB200_LARGE_N=28: every block that is not stored takes the large paths
  control  no switch: the same jobs on the pooled path
  edge     BSCB200_LARGE_N=100000: a block of 100000 bytes stays on the pooled path, one of 100001 bytes is routed

The parent computes every expected output on the CPU: the reference (oracle/_ref) for sorters 1 and 3..6, LZP and in-place blocks, the C
port for ST7 and ST8, and the known answer K5 of SURVEY.md.  With BSCB200_STSTATS=1 the lean inverse ST prints the list count of every
block; it must equal st_lists() of the block's text, which proves that the lean path ran and checks its dynamic-group classification.
The pooled path prints no such line."""
import copy
import ctypes
import re
import zlib

import numpy as np
import pytest

import reference_inputs as ri
import test_gpu_parity as tp
import test_oracle as to
from test_gpu_pipeline import Battery, compare, run_child

MIB = 1 << 20
SLACK = 64 * MIB                         # free HBM at the end of a child is within this of its value after the first routed calls
EDGE_SIZES = [255, 256, 257, 261, 262, 263, 2047, 2048, 2049, 4095, 4096, 4097, 6143, 6144, 6145, 8191, 8192, 8193, 65535, 65536, 65537]
LZP_SETTINGS = [(15, 128), (12, 4), (18, 255)]
SWEEP_SORTERS = (1, 3, 4, 5, 6, 7, 8)
K5 = dict(seed=3, n=33554432, size=32294018, adler32=0x8D12E56B)    # SURVEY.md known answer: 32 MiB skew, ST6, coder 1
EDGE_N = 100000
STSTATS = re.compile(r"\[ststats\] n (\d+) k (\d) lists (\d+)")
vp = ctypes.c_void_p


# ---- the list count of the inverse ST ------------------------------------------------------------------------------------------
def st_lists(T, k):
    """The number of lists st_serial walks when it inverts the order-k ST of T: the occurrences of every k-gram of T (read cyclically)
    that is followed by at least two distinct bytes, plus 1 if the k-gram at position 0 is not one of those."""
    T = np.ascontiguousarray(T, dtype=np.uint8)
    n = T.size
    ext = np.tile(T, (k + 1) // n + 2) if n <= k else np.concatenate([T, T[:k + 1]])
    key = np.zeros(n, dtype=np.uint64)
    for c in range(k):
        key = (key << np.uint64(8)) | ext[c:c + n]
    nxt = ext[k:k + n]
    if k <= 7:                                              # k-gram and next byte in one u64
        s = np.sort((key << np.uint64(8)) | nxt)
        sk, sn = s >> np.uint64(8), (s & np.uint64(255)).astype(np.uint8)
    else:
        o = np.argsort(key, kind="stable")
        sk, sn = key[o], nxt[o]
    start = np.flatnonzero(np.r_[True, sk[1:] != sk[:-1]])
    dynamic = np.minimum.reduceat(sn, start) != np.maximum.reduceat(sn, start)
    count = np.diff(np.r_[start, n])
    first = int(np.searchsorted(sk[start], key[0]))
    return int(count[dynamic].sum()) + (0 if dynamic[first] else 1)


def kernel_heads(T, k):
    """A numpy model of how the inverse ST picks the heads of its lists: the order-k ST of T, LF, the k-groups (st_round), the dynamic
    flag of each group (st_groups: the LF-image of its first and last row fall in different (k - 1)-groups) and the heads
    h == index || dynf[gk[h]].  Returns (number of heads, whether the k-gram at position 0 is dynamic)."""
    T = np.ascontiguousarray(T, dtype=np.uint8)
    n = T.size
    keys = T[(np.arange(n)[:, None] + np.arange(k)[None, :]) % n]
    order = np.lexsort(tuple(keys[:, c] for c in range(k - 1, -1, -1)))    # stable: rows of equal k-grams keep their text order
    L = T[(order - 1) % n]
    index = int(np.flatnonzero(order == 0)[0])
    rk = keys[order]
    LF = np.empty(n, dtype=np.int64)
    LF[np.argsort(L, kind="stable")] = np.arange(n)
    new_group = np.ones(n, dtype=bool)
    new_group[1:] = np.any(rk[1:] != rk[:-1], axis=1)
    gk = np.maximum.accumulate(np.where(new_group, np.arange(n), 0))
    tmpk = np.empty(n, dtype=np.int64)
    tmpk[LF] = gk
    last = np.ones(n, dtype=bool)
    last[:-1] = gk[1:] != gk[:-1]
    dynf = np.zeros(n, dtype=bool)
    for j in np.flatnonzero(last):
        dynf[gk[j]] = tmpk[gk[j]] != tmpk[j]
    heads = dynf[gk] | (np.arange(n) == index)
    return int(heads.sum()), bool(dynf[gk[index]])


def adler32(a):
    return zlib.adler32(memoryview(np.ascontiguousarray(a, dtype=np.uint8)))


def block_mode(blk):
    return int(np.asarray(blk[8:12], dtype=np.uint8).view("<u4")[0])


# ---- the battery ---------------------------------------------------------------------------------------------------------------
def decode_cases(gen, big=True):
    """(name, input, sorter, coder, lzp) of every reference block the decode battery restores; `big` adds the 64 MiB and K5 blocks"""
    for name, a in tp.small_inputs(gen):
        for s in (3, 4, 5, 6, 7, 8):
            for c in (1, 2, 3):
                yield "%s/m%de%d" % (name, s, c), a, s, c, None
    for i, (name, a) in enumerate(to._sweep_inputs(160, 20260924)):
        if a.size <= 28:                                    # stored blocks
            continue
        s, c = SWEEP_SORTERS[i % 7], 1 + i % 3
        lzp = LZP_SETTINGS[(i // 5) % 3] if i % 5 == 0 and s <= 6 else None
        yield "%s/m%de%d%s" % (name, s, c, "/lzp%d,%d" % lzp if lzp else ""), a, s, c, lzp
    for name, a in ri.lzp_inputs(gen).items():
        for lzp in LZP_SETTINGS:
            for c in (1, 3):
                for s in (1, 6):
                    yield "lzp %s/m%de%d/lzp%d,%d" % (name, s, c, lzp[0], lzp[1]), a, s, c, lzp
    rng = np.random.default_rng(262)
    j = 0
    for n in EDGE_SIZES:
        for kind, a in (("text", gen.text(n % 89 + 1, n)), ("skew", gen.skew(n % 83 + 1, n)), ("alpha2", rng.integers(0, 2, n, dtype=np.uint8))):
            for _ in range(2):
                s, c = 3 + j % 6, 1 + j % 3
                j += 1
                yield "edge %s n=%d/m%de%d" % (kind, n, s, c), a, s, c, None
    if big:
        for name, a in ri.degenerate_inputs().items():
            yield "64M %s/m6e1" % name, a, 6, 1, None
        yield "K5 skew 32M/m6e1", gen.skew(K5["seed"], K5["n"]), 6, 1, None


def reference_block(ref, port, a, s, c, lzp):
    if lzp:
        return ref.compress_lzp(a, lzp[0], lzp[1], s, c, 3)
    return (port if s >= 7 else ref).compress(a, s, c, 3)  # ST7 and ST8 exist only in the reference's CUDA build


def ref_inplace(ref, a, s, c, f, lzp=None):
    """the reference's in-place bsc_compress; on failure the expected buffer is the caller's, untouched (n + 92 bytes, as the child's)"""
    n = a.size
    buf = np.zeros(n + 28 + 64, dtype=np.uint8)
    buf[:n] = a
    h, m = lzp or (0, 0)
    r = ref.lib.bsc_compress(vp(buf.ctypes.data), vp(buf.ctypes.data), n, h, m, s, c, f)
    return r, (buf[:r].copy() if r > 0 else untouched(a))


def untouched(a):
    """the buffer of an in-place compress job as the caller filled it"""
    buf = np.zeros(a.size + 28 + 64, dtype=np.uint8)
    buf[:a.size] = a
    return buf


def sentinel(a, n):
    """what a raw_decompress job returns: the output, then 64 bytes of 0xA5; all 0xA5 when a is None (a call that must write nothing)"""
    out = np.full(n + 64, 0xA5, dtype=np.uint8)
    if a is not None:
        out[:n] = a
    return out


class LargeBattery(Battery):
    def __init__(self, root, name):
        super().__init__(root, name)
        self.lists = {}                                     # job name: (n, k, list count or None) of every ST block

    def decode(self, name, blk, a, lists=None):
        """one block, out of place into a sentinel-filled buffer and in place; `lists`: the list count of its ST, if known"""
        n, mode = a.size, block_mode(blk)
        self.add(name + " raw", "raw_decompress", blk, (0, sentinel(a, n)), dict(n=n))
        self.add(name + " inplace", "inplace_decompress", blk, (0, a), dict(n=n))
        if (mode & 0x1F) >= 3:
            self.lists[name + " raw"] = self.lists[name + " inplace"] = (n, mode & 0x1F, lists)


@pytest.fixture(scope="module")
def decode_jobs(tmp_path_factory, gen, ref, port):
    bat = LargeBattery(tmp_path_factory.mktemp("large_dec"), "dec")
    lists = {}                                              # (input, k): list count; an input's name is the case's up to "/"
    for i, (name, a, s, c, lzp) in enumerate(decode_cases(gen)):
        z, blk = reference_block(ref, port, a, s, c, lzp)
        assert z > 0, (name, z)
        if name.startswith("K5"):
            assert z == K5["size"] and adler32(blk) == K5["adler32"], "K5: the reference's block differs from SURVEY.md's"
        mode, count = block_mode(blk), None
        if (mode & 0x1F) >= 3 and (mode >> 8) == 0:        # an ST block without LZP: its text is the input
            key = (name.split("/")[0], mode & 0x1F)
            if key not in lists:
                lists[key] = st_lists(a, mode & 0x1F)
            count = lists[key]
        bat.decode(name, blk, a, count)
        if i == 20:                                         # every coder and ST3..ST8 have run: kernel images are loaded
            bat.add("hbm after the first calls", "free_hbm", np.zeros(1, np.uint8), (0, None))
    # corrupt ST blocks: L is random, so its lists do not tile a text; header and payload checksums are right
    rng = np.random.default_rng(5)
    for n in (1000, 70000, 1 << 20):
        L = rng.integers(0, 7, n, dtype=np.uint8)
        r, payload = ref.coder_compress(L, 1, 3)
        assert r > 0
        for s in (3, 6):
            h = np.zeros(28, dtype=np.uint8)
            h[0:24].view("<u4")[:] = [28 + r, n, s | (1 << 5), int(rng.integers(0, n)), adler32(L), adler32(payload)]
            h[24:28].view("<u4")[0] = adler32(h[:24])
            name = "corrupt L n=%d/m%de1" % (n, s)
            bat.add(name, "raw_decompress", np.concatenate([h, payload]), (-6, sentinel(None, n)), dict(n=n))
            bat.lists[name] = (n, s, None)
    bat.add("hbm at the end", "free_hbm", np.zeros(1, np.uint8), (0, None))
    return bat


@pytest.fixture(scope="module")
def compress_jobs(tmp_path_factory, gen, ref):
    """In-place bsc_compress (compress_large when routed), and out-of-place calls above the threshold, which must stay on the pooled path.
    The inputs have 65536 bytes or more.  Below that the reference drops the secondary indexes (libbsc.cpp:303), and so does the pooled
    path, but compress_large keeps them: in production it never sees a block that small."""
    bat = Battery(tmp_path_factory.mktemp("large_comp"), "comp")
    bat.control = {}                                        # job name: what the pooled path returns where it differs
    inputs = {"text100k": gen.text(3, 100000), "skew200k": gen.skew(4, 200000), "rep700x200": np.tile(gen.text(3, 700), 200)}
    inputs.update({name: a for name, (a, s) in ri.inplace_inputs(gen).items() if s == 1})
    for i, (name, a) in enumerate(inputs.items()):
        for c in (1, 2, 3):
            for f in (1, 3):
                for lzp in (None, (15, 128)):
                    want = ref_inplace(ref, a, 1, c, f, lzp)
                    assert want[0] > 0, (name, c, f, lzp)
                    bat.add("inplace %s/m1e%d f%d%s" % (name, c, f, " lzp" if lzp else ""), "compress", a, want,
                            dict(sorter=1, coder=c, features=f, lzp=list(lzp or (0, 0)), inplace=True))
        if i == 0:
            bat.add("hbm after the first calls", "free_hbm", np.zeros(1, np.uint8), (0, None))
    a = gen.rand(1, 300000)
    for lzp in (None, (15, 128)):                           # LZP does not shrink random data: the block goes on without it
        want = ref_inplace(ref, a, 1, 1, 3, lzp)
        assert want[0] == -3
        bat.add("inplace rand300k%s" % (" lzp" if lzp else ""), "compress", a, want,
                dict(sorter=1, coder=1, features=3, lzp=list(lzp or (0, 0)), inplace=True))
    for name, (a, s) in ri.inplace_inputs(gen).items():    # the forward ST has no bounded variant: LIBBSC_NOT_SUPPORTED, buffer untouched
        if s != 1:
            job = "inplace %s/m%de1" % (name, s)
            bat.add(job, "compress", a, (-4, untouched(a)), dict(sorter=s, coder=1, features=3, inplace=True))
            bat.control[job] = ref_inplace(ref, a, s, 1, 3)
    for name, a in (("text5_300k", ri.inplace_inputs(gen)["text5_300k"][0]), ("skew200k", inputs["skew200k"])):
        for s, c in ((1, 2), (6, 3)):
            bat.add("out of place %s/m%de%d" % (name, s, c), "compress", a, ref.compress(a, s, c, 3), dict(sorter=s, coder=c, features=3))
        bat.add("out of place %s/m1e1 lzp12,4" % name, "compress", a, ref.compress_lzp(a, 12, 4, 1, 1, 3),
                dict(sorter=1, coder=1, features=3, lzp=[12, 4]))
    bat.add("hbm at the end", "free_hbm", np.zeros(1, np.uint8), (0, None))
    return bat


@pytest.fixture(scope="module")
def edge_jobs(tmp_path_factory, gen, ref):
    """blocks of EDGE_N and EDGE_N + 1 bytes under BSCB200_LARGE_N=EDGE_N: only the second is routed"""
    bat = LargeBattery(tmp_path_factory.mktemp("large_edge"), "edge")
    for n in (EDGE_N, EDGE_N + 1):
        a = gen.text(5, n)
        for s in (1, 6):
            bat.decode("text n=%d/m%de1" % (n, s), ref.compress(a, s, 1, 3)[1], a, st_lists(a, s))
            want = (-4, untouched(a)) if n > EDGE_N and s != 1 else ref_inplace(ref, a, s, 1, 3)
            bat.add("inplace text n=%d/m%de1" % (n, s), "compress", a, want, dict(sorter=s, coder=1, features=3, inplace=True))
    return bat


# ---- checks --------------------------------------------------------------------------------------------------------------------
def env(threshold):
    """the child's switches: BSCB200_LARGE_N set to `threshold`, or to nothing (the default) for None"""
    return {"BSCB200_LARGE_N": "" if threshold is None else str(threshold), "BSCB200_STSTATS": "1"}


def outputs(bat, results, d, config):
    """compare()'s findings as a list, so that a test can report them together with the list counts"""
    try:
        compare(bat, results, d, config)
    except AssertionError as e:
        return [str(e)]
    return []


def check_lists(bat, per_job, threshold):
    """Every ST block above `threshold` (None: no block) printed one [ststats] line with its order and, where the battery knows it, its
    list count; every other job printed none.  Returns the findings and how many list counts were compared."""
    bad, checked = [], 0
    for job in bat.jobs:
        name = job["name"]
        lines = [m for m in (STSTATS.search(line) for line in per_job.get(name, [])) if m]
        n, k, want = bat.lists.get(name, (0, 0, None))
        if not (k and threshold is not None and n > threshold):
            if lines:
                bad.append("%s: the lean inverse ST ran (%s)" % (name, lines[0].group(0)))
            continue
        if len(lines) != 1:
            bad.append("%s: %d [ststats] lines, not one: the lean inverse ST did not run" % (name, len(lines)))
            continue
        got_n, got_k, got = (int(x) for x in lines[0].groups())
        if got_k != k or (want is not None and (got_n, got) != (n, want)):
            bad.append("%s: lean inverse ST of n %d k %d walked %d lists; the text has n %d k %d and %s lists" % (name, got_n, got_k, got, n, k, want))
        checked += want is not None
    return bad, checked


def free_is_back(results, config):
    first, last = results["hbm after the first calls"]["free"], results["hbm at the end"]["free"]
    assert abs(first - last) <= SLACK, "%s: %d bytes of HBM free after the first calls, %d at the end" % (config, first, last)


# ---- GPU -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_routed_decode(bsc, decode_jobs):
    """Every block of the battery through the large paths: output, in place and into a sentinel-filled buffer, the lean path's list
    counts, LIBBSC_DATA_CORRUPT with nothing written for the corrupt blocks, and no HBM kept per call."""
    results, _, per_job, d = run_child(decode_jobs, "routed decode", env(28), timeout=1800)
    bad = outputs(decode_jobs, results, d, "routed decode")
    lists, checked = check_lists(decode_jobs, per_job, 28)
    assert not bad and not lists, "\n".join(bad + ["lists:"] + lists[:20])
    assert checked >= 750, checked
    free_is_back(results, "routed decode")


@pytest.mark.gpu
def test_control_decode(bsc, decode_jobs):
    results, _, per_job, d = run_child(decode_jobs, "control decode", env(None), timeout=1800)
    compare(decode_jobs, results, d, "control decode")
    lists, _ = check_lists(decode_jobs, per_job, None)
    assert not lists, "\n".join(lists[:20])


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["routed", "control"])
def test_inplace_compress(bsc, compress_jobs, config):
    bat = compress_jobs
    if config == "control":
        bat = copy.copy(bat)
        bat.expect = dict(bat.expect, **bat.control)
    results, _, _, d = run_child(bat, "compress " + config, env(28 if config == "routed" else None))
    compare(bat, results, d, "compress " + config)
    free_is_back(results, "compress " + config)


@pytest.mark.gpu
def test_threshold_edge(bsc, edge_jobs):
    results, _, per_job, d = run_child(edge_jobs, "edge", env(EDGE_N))
    compare(edge_jobs, results, d, "edge")
    lists, checked = check_lists(edge_jobs, per_job, EDGE_N)
    assert not lists and checked == 2, (lists, checked)


# ---- CPU -----------------------------------------------------------------------------------------------------------------------
def test_list_formula_matches_the_head_selection():
    rng = np.random.default_rng(1)
    for t in range(300):
        n, sigma, k = int(rng.integers(2, 300)), int(rng.choice([1, 2, 3, 4, 16])), int(rng.integers(3, 9))
        T = rng.integers(0, sigma, n, dtype=np.uint8)
        if t % 3 == 0:                                      # periodic
            p = T[:max(1, n // 7)]
            T = np.tile(p, n // p.size + 1)[:n]
        assert kernel_heads(T, k)[0] == st_lists(T, k), (t, n, sigma, k)


def st_cases(gen, limit):
    return [(name, a, s) for name, a, s, c, lzp in decode_cases(gen, big=False) if s >= 3 and lzp is None and a.size <= limit]


def test_battery_has_both_kinds_of_position_0(gen):
    """the k-gram at position 0 is dynamic in some ST block of the battery and static in another"""
    seen = {}
    for name, a, s in st_cases(gen, 8193):
        seen.setdefault(kernel_heads(a, s)[1], name)
        if len(seen) == 2:
            break
    assert set(seen) == {True, False}, seen


def test_battery_has_one_list_and_more_than_half(gen):
    counts = {name: (st_lists(a, s), a.size) for name, a, s in st_cases(gen, 70000)}
    assert counts["zeros1000/m3e1"] == (1, 1000)
    assert any(x > n // 2 for x, n in counts.values()), counts


def test_battery_has_every_edge_size(gen):
    have = {(name.split()[1], a.size) for name, a, s, c, lzp in decode_cases(gen, big=False) if name.startswith("edge ")}
    assert have == {(kind, n) for kind in ("text", "skew", "alpha2") for n in EDGE_SIZES}
    assert {a.size for name, a, s, c, lzp in decode_cases(gen, big=False)} >= set(EDGE_SIZES)
