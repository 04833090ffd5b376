"""The staged rank and L stores of the standard forward BWT (csrc/bwt_encode.cu): bwt_apply and bwt_emit write (value, position)
pairs, one radix pass partitions them by position window, and bwt_stage_scatter stores them window after window.
BSCB200_BWT_STAGE=<0|1> forces the direct or the staged store for one process, so each setting runs in a child of its own
(tests/gpu_child.py):

  stage=1 with BSCB200_BWT_SEG = 0, 1 and 256    every split and the emit staged, under each round sort
  stage=0                                        every store direct (the path before the staged one)
  unset                                          the size threshold picks per split

Every setting must give the reference's index, secondary indexes, L and compressed block on n = 1..300, on n around the radix digit
boundaries (2^k - 1, 2^k, 2^k + 1 for k = 8..26) and on 1-8 MiB text, skew, random, two-letter and long-run blocks, and the settings
must agree with each other there; the 64 MiB zero, period-7 and period-8 blocks, staged, must give their golden digests.  The profile
shows which store ran."""
import json
import os

import numpy as np
import pytest

import reference_inputs as ri
from test_gpu_pipeline import Battery, compare, run_child
from test_gpu_segmented_bwt import same_as

pytestmark = pytest.mark.gpu

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_results.json")))
SETTINGS = [("stage=1 seg=0", {"BSCB200_BWT_STAGE": "1", "BSCB200_BWT_SEG": "0"}),
            ("stage=1 seg=1", {"BSCB200_BWT_STAGE": "1", "BSCB200_BWT_SEG": "1"}),
            ("stage=1 seg=256", {"BSCB200_BWT_STAGE": "1", "BSCB200_BWT_SEG": "256"}),
            ("stage=0", {"BSCB200_BWT_STAGE": "0"}),
            ("default", {})]
STAGED = ("bwt_apply_staged", "bwt_stage_rank", "bwt_emit_staged", "bwt_stage_L")


def blocks(gen):
    """1-8 MiB blocks of each kind"""
    rng = np.random.default_rng(20261019)
    out = []
    for i, mib in enumerate((1, 3, 8)):
        n = (mib << 20) + 17 * i
        out += [("text %d MiB" % mib, gen.text(i + 2, n)), ("skew %d MiB" % mib, gen.skew(i + 2, n)),
                ("random %d MiB" % mib, gen.rand(i + 2, n)),
                ("alphabet-2 %d MiB" % mib, rng.integers(0, 2, n, dtype=np.uint8) + 97),
                ("long runs %d MiB" % mib, np.repeat(rng.integers(0, 4, n // 1000 + 1, dtype=np.uint8), rng.integers(1, 2000, n // 1000 + 1))[:n])]
    return out


def reference_bwt(checker, a):
    """the reference's (index, L, secondary indexes); below 16 bytes, where no secondary index can be asked for, only the other
    settings are the yardstick"""
    if a.size < 16:
        return (None, None)
    r, L, aux = checker.bwt_encode(a)
    return (r, L, list(aux))


@pytest.fixture(scope="module")
def battery(tmp_path_factory, gen, checker):
    bat = Battery(tmp_path_factory.mktemp("staged"), "staged")
    for n in range(1, 301):
        a = gen.text(n % 7 + 1, n)
        bat.add("n=%d" % n, "bwt_encode", a, reference_bwt(checker, a))
    for k in range(8, 27):
        for n in ((1 << k) - 1, 1 << k, (1 << k) + 1):
            a = gen.text(k, n)
            bat.add("n=%d" % n, "bwt_encode", ("text", k, n), reference_bwt(checker, a))
    for name, a in blocks(gen):
        bat.add(name, "bwt_encode", a, reference_bwt(checker, a))
        z, blk = checker.compress(a, 1, 1, 3)
        bat.add(name + " compressed", "compress", a, (z, blk), dict(sorter=1, coder=1, features=3))
    bat.add("profile text1M", "bwt_profiled", gen.text(2, 1 << 20), (None, None))
    return bat


@pytest.fixture(scope="module")
def children(battery):
    return {config: run_child(battery, config, env, timeout=1800) for config, env in SETTINGS}


@pytest.mark.parametrize("config", [c for c, _ in SETTINGS])
def test_staged_scatter_matches_reference(battery, children, config):
    results, _, _, d = children[config]
    saved, battery.expect = battery.expect, {name: exp for name, exp in battery.expect.items() if exp[0] is not None}
    try:
        compare(battery, results, d, config)
    finally:
        battery.expect = saved
    first = SETTINGS[0][0]
    r0, _, _, d0 = children[first]
    bad = same_as(battery, results, d, r0, d0, [n for n in battery.expect if n != "profile text1M"])
    assert not bad, (config, "differs from", first, bad[:10])
    prof = results["profile text1M"]["profile"]
    env = dict(SETTINGS)[config]
    if env.get("BSCB200_BWT_STAGE") == "1":
        assert all(k in prof for k in STAGED), sorted(prof)
        assert "bwt_emit" not in prof, sorted(prof)
    elif env.get("BSCB200_BWT_STAGE") == "0":
        assert not any(k in prof for k in STAGED), sorted(prof)


def test_staged_scatter_64MiB_degenerate(tmp_path_factory):
    """the 64 MiB zero, period-7 and period-8 blocks, every store staged: L, indexes and compressed block against the golden digests"""
    bat = Battery(tmp_path_factory.mktemp("staged_big"), "big")
    for name in ("zeros", "period7", "period8"):
        want = GOLD["degenerate"][name]
        bat.add(name, "bwt_encode", ("degenerate", name, 0), (want["index"], want["L"], want["aux"]))
        bat.add(name + " compressed", "compress", ("degenerate", name, 0), (want["block"]["size"], want["block"]),
                dict(sorter=1, coder=1, features=3))
    results, _, _, d = run_child(bat, "stage=1", {"BSCB200_BWT_STAGE": "1"}, timeout=1800)
    compare(bat, results, d, "stage=1")
