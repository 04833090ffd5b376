"""The segmented doubling rounds of the forward BWT (csrc/bwt_encode.cu): groups of at most S entries sorted inside one CTA, the
larger ones compacted and radix-sorted.  BSCB200_BWT_SEG=<S> sets the bound for one process, so each setting runs in a child of its own
(tests/gpu_child.py):

  default   no switch: S = 256
  0         every group through the global radix sort (the path before the split)
  1         every group is large: compaction, radix sort and scatter alone
  2, 33     small bounds put group-size edges and CTA boundaries into small inputs
  255, 257  the default's S - 1 and S + 1
  1024      the largest bound (SEG_MAX)

Every setting must give the reference's index, secondary indexes and L on the parity inputs, the seeded sweep, n = 1..300 at unaligned
device addresses and crafted texts whose h = 8 round has groups of exactly S - 1, S and S + 1 entries for each S above; the golden
digests on the 64 MiB degenerate blocks; and the switch-0 output on a 64 MiB text block.  The profile shows which path ran."""
import json
import os
import time

import numpy as np
import pytest

import reference_inputs as ri
import test_gpu_parity as tp
from test_gpu_pipeline import Battery, compare, run_child
from test_oracle import _sweep_inputs

pytestmark = pytest.mark.gpu

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_results.json")))
SETTINGS = [None, 0, 1, 2, 33, 255, 257, 1024]
BOUNDS = [1, 2, 33, 256, 1024]                      # the S whose S - 1, S and S + 1 groups the crafted texts hold
BIG_S = 30                                          # seconds per 64 MiB block


def crafted(S, seed):
    """A text whose 8-byte prefixes are unique except for markers: marker k (bytes >= 200, first byte unique) occurs c_k times, each
    followed by random bytes, so the h = 8 round has one group of exactly c_k entries per marker with distinct key2.  The counts are
    S - 1, S and S + 1, then counts around them, so that groups of many sizes follow each other and straddle CTA slot ranges."""
    rng = np.random.default_rng(seed)
    counts = [c for c in (S - 1, S, S + 1) if c >= 2] + [int(x) for x in rng.integers(2, S + 3, 40)]
    pieces = []
    for k, c in enumerate(counts):
        marker = np.array([200 + k % 50, 250, 251, 252, 253, 254, 255, k // 50], dtype=np.uint8)
        for _ in range(c):
            pieces.append(np.concatenate([marker, rng.integers(0, 200, int(rng.integers(8, 24)), dtype=np.uint8)]))
    pieces += [rng.integers(0, 200, int(rng.integers(8, 64)), dtype=np.uint8) for _ in range(len(pieces) // 2)]
    order = rng.permutation(len(pieces))
    return np.concatenate([pieces[i] for i in order])


def reference(checker, a):
    """the reference's (index, L, secondary indexes); below 16 bytes, where no secondary index can be asked for, only the switch-0
    output is the yardstick"""
    if a.size < 16:
        return (None, None)
    r, L, aux = checker.bwt_encode(a)
    return (r, L, list(aux))


@pytest.fixture(scope="module")
def battery(tmp_path_factory, gen, checker):
    bat = Battery(tmp_path_factory.mktemp("seg_bwt"), "seg")
    inputs = [("parity " + name, a) for name, a in tp.small_inputs(gen)]
    inputs += [("sweep %d" % i, a) for i, (_, a) in enumerate(_sweep_inputs(160, 20260924))]
    inputs += [("crafted S=%d seed=%d" % (S, s), crafted(S, 100 * S + s)) for S in BOUNDS for s in (1, 2)]
    for name, a in inputs:
        bat.add(name, "bwt_encode", a, reference(checker, a))
    for n in range(1, 301):                         # device pointers at offsets 0, 1 and 7 from a 256-byte boundary
        a = gen.text(n % 7 + 1, n)
        bat.add("n=%d unaligned" % n, "device_guarded", a, reference(checker, a), dict(call="bwt_encode"))
    bat.add("profile text1M", "bwt_profiled", gen.text(2, 1 << 20), (None, None))
    return bat


@pytest.fixture(scope="module")
def big(tmp_path_factory):
    bat = Battery(tmp_path_factory.mktemp("seg_bwt_big"), "big")
    for name in ri.degenerate_inputs():
        want = GOLD["degenerate"][name]
        bat.add("degenerate " + name, "bwt_encode", ("degenerate", name, 0), (want["index"], want["L"], want["aux"]))
    bat.add("text 64MiB", "bwt_encode", ("text", 2, 64 << 20), (None, None))
    return bat


def env(S):
    """the child's switch; for the default, the variable is not set at all"""
    return {} if S is None else {"BSCB200_BWT_SEG": str(S)}


def same_as(bat, results, d, other, other_d, names):
    """outputs of `names` equal in two children's results"""
    bad = []
    for name in names:
        a, b = results[name], other[name]
        la = np.load(os.path.join(d, "out", bat.files[name] + ".npy"))
        lb = np.load(os.path.join(other_d, "out", bat.files[name] + ".npy"))
        if a["r"] != b["r"] or a.get("aux") != b.get("aux") or not np.array_equal(la, lb):
            bad.append(name)
    return bad


@pytest.fixture(scope="module")
def switch0(battery, big):
    return run_child(battery, "seg=0", env(0)), run_child(big, "seg=0", env(0), timeout=1800)


@pytest.mark.parametrize("S", SETTINGS, ids=lambda s: "default" if s is None else str(s))
def test_segmented_bwt_matches_reference(battery, switch0, S):
    config = "seg=%s" % S
    results, _, _, d = switch0[0] if S == 0 else run_child(battery, config, env(S))
    checked = {name: exp for name, exp in battery.expect.items() if exp[0] is not None}
    saved, battery.expect = battery.expect, checked
    try:
        compare(battery, results, d, config)
    finally:
        battery.expect = saved
    for name in battery.expect:
        rec = results[name]
        if "guards" in rec:
            assert all(rec["guards"]) and rec["offsets_agree"], (config, name, rec["codes"], rec["guards"])
    if S != 0:
        r0, _, _, d0 = switch0[0]
        bad = same_as(battery, results, d, r0, d0, [n for n in battery.expect if n != "profile text1M"])
        assert not bad, (config, bad[:10])
    prof = results["profile text1M"]["profile"]
    seg = sorted(k for k in prof if k.startswith("bwt_seg_"))
    if S == 0:
        assert not seg, seg
    else:
        assert "bwt_seg_count" in prof and "bwt_seg_starts" in prof, seg
        assert ("bwt_seg_sort" in prof) == (S != 1), seg             # at S = 1 every group is large
        assert ("bwt_seg_compact" in prof) == (S == 1 or "bwt_seg_scatter" in prof), seg


@pytest.mark.parametrize("S", SETTINGS, ids=lambda s: "default" if s is None else str(s))
def test_segmented_bwt_64MiB(big, switch0, S):
    """the degenerate blocks against their golden digests, and a text block against the switch-0 output, within BIG_S per block"""
    config = "seg=%s" % S
    t0 = time.time()
    results, _, _, d = switch0[1] if S == 0 else run_child(big, config, env(S), timeout=1800)
    dt = time.time() - t0
    saved, big.expect = big.expect, {k: v for k, v in big.expect.items() if v[0] is not None}
    try:
        compare(big, results, d, config)
    finally:
        big.expect = saved
    if S != 0:
        r0, _, _, d0 = switch0[1]
        assert not same_as(big, results, d, r0, d0, list(big.expect)), config
        assert dt < BIG_S * len(big.expect) + 60, (config, dt)                # + the child's start and the inputs' generation
