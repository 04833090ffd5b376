"""The `bsc1` file container and the block scheduler of libbsc_b200/cli/bsc_b200.cpp (SURVEY.md 8f #3).

CPU part: the same CLI source is built against the UNMODIFIED reference library (-DBSCB200_CLI_REF: identical block API, no
GPU) and its archives are compared with the reference's own CLI (oracle/_ref/bsc, built by oracle/Makefile from the
reference's bsc.cpp): byte-identical containers when both write blocks in order (`bsc -t`), and each side decodes the
other's archives.  That pins the container logic, option handling and the in-order writer without a GPU.
GPU part: the product binary libbsc_b200/bsc_b200 round-trips a file and produces the bytes of the reference CLI (its
archive's size and SHA-256, tests/golden/reference_results.json)."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import reference_inputs as ri

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "libbsc_b200", "cli", "bsc_b200.cpp")
REFDIR = os.path.join(ROOT, "oracle", "_ref")
REFCLI = os.path.join(REFDIR, "bsc")
TESTCLI = os.path.join(ROOT, "tools", "bin", "bsc_b200_ref")
PRODUCT = os.path.join(ROOT, "libbsc_b200", "bsc_b200")


def _run(*cmd):
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, (cmd, p.stdout[-300:], p.stderr[-300:])
    return p.stdout


@pytest.fixture(scope="module")
def clis(tmp_path_factory):
    if not (os.path.exists(REFCLI) and os.path.exists(os.path.join(REFDIR, "libbsc_ref.so"))):
        pytest.skip("oracle/_ref (reference library + CLI) not built")
    os.makedirs(os.path.dirname(TESTCLI), exist_ok=True)
    if not os.path.exists(TESTCLI) or os.path.getmtime(SRC) > os.path.getmtime(TESTCLI):
        _run("/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-pthread", "-fopenmp", "-DBSCB200_CLI_REF", SRC, "-o", TESTCLI,
             "-L" + REFDIR, "-lbsc_ref", "-Wl,-rpath," + REFDIR)
    return tmp_path_factory.mktemp("cli")


def _files(gen, d):
    rng = np.random.default_rng(3)
    cases = {"text3M": gen.text(2, 3 << 20), "ragged": gen.text(5, (1 << 20) + 12345), "rand": gen.rand(1, 300000),
             "tiny": gen.text(1, 20), "empty": np.zeros(0, np.uint8), "skew": gen.skew(3, 2 << 20),
             "runs": np.repeat(rng.integers(0, 50, 4000, dtype=np.uint8), rng.integers(1, 2000, 4000))[: 3 << 20]}
    out = {}
    for name, a in cases.items():
        p = str(d / (name + ".bin"))
        a.tofile(p)
        out[name] = p
    return out


def test_container_matches_reference_cli(clis, gen):
    d = clis
    for name, path in _files(gen, d).items():
        for opts in (["-b1"], ["-b1", "-m5"], ["-b2", "-e0"], ["-b1", "-e2"]):
            ours, theirs = str(d / "ours.bsc"), str(d / "theirs.bsc")
            _run(TESTCLI, "e", path, ours, *opts, "-j3")
            _run(REFCLI, "e", path, theirs, *opts, "-p", "-t")
            a, b = open(ours, "rb").read(), open(theirs, "rb").read()
            assert a == b, (name, opts, len(a), len(b))
            if "-m5" in opts:
                continue                                           # ST decoding stays in the reference (DESIGN.md 1)
            back1, back2 = str(d / "back1.bin"), str(d / "back2.bin")
            _run(TESTCLI, "d", theirs, back1, "-j2")                   # their archive, our reader
            _run(REFCLI, "d", ours, back2)                             # our archive, their reader
            orig = open(path, "rb").read()
            assert open(back1, "rb").read() == orig and open(back2, "rb").read() == orig, (name, opts)


def test_reader_accepts_blocks_in_any_order(clis, gen):
    """The reference writes blocks in completion order when it runs multithreaded (bsc.cpp:398-417)."""
    d = clis
    path = str(d / "mt.bin")
    gen.text(9, 6 << 20).tofile(path)
    arch, back = str(d / "mt.bsc"), str(d / "mt.back")
    _run(REFCLI, "e", path, arch, "-b1", "-p")                          # parallel block loop of the reference
    _run(TESTCLI, "d", arch, back, "-j4")
    assert open(back, "rb").read() == open(path, "rb").read()


def test_reader_accepts_reference_default_archives(clis, gen):
    """`bsc e in out` (LZP on, parallel block loop): the container carries LZP blocks, the block API undoes them."""
    d = clis
    path = str(d / "dflt.bin")
    np.tile(gen.text(8, 300000), 12).tofile(path)                       # repetitive: LZP finds matches
    arch, back = str(d / "dflt.bsc"), str(d / "dflt.back")
    _run(REFCLI, "e", path, arch, "-b1")
    _run(TESTCLI, "d", arch, back, "-j3")
    assert open(back, "rb").read() == open(path, "rb").read()


def test_lzp_option_matches_reference_default(clis, gen):
    """`bsc_b200 e -l` = `bsc e` (LZP 15 / 128 on, filters off); `-H` / `-M` as in bsc."""
    d = clis
    path = str(d / "l.bin")
    np.tile(gen.text(8, 300000), 12).tofile(path)
    for ours_opts, their_opts in ((["-l"], []), (["-l", "-H16", "-M64"], ["-H16", "-M64"]), (["-M200"], ["-M200"])):
        ours, theirs = str(d / "l_ours.bsc"), str(d / "l_theirs.bsc")
        _run(TESTCLI, "e", path, ours, "-b1", "-j3", *ours_opts)
        _run(REFCLI, "e", path, theirs, "-b1", "-t", *their_opts)
        assert open(ours, "rb").read() == open(theirs, "rb").read(), ours_opts


def test_reader_undoes_reference_filters(clis, gen):
    """Archives made with the reference's host-side filters: reversed contexts (-cp), autodetected contexts (-ca), record
    reordering (-r) and segmentation (-s).  The inverse filters are applied after the blocks are decoded."""
    d = clis
    rng = np.random.default_rng(8)
    recs = np.zeros((300000, 4), dtype=np.uint8)                        # 4-byte records: slowly varying columns -> the detector picks recordSize 4
    recs[:, 0] = np.arange(300000) & 255; recs[:, 1] = (np.arange(300000) >> 8) & 255; recs[:, 2] = 7; recs[:, 3] = rng.integers(0, 3, 300000)
    files = {"text": gen.text(4, (1 << 20) + 77), "records": recs.reshape(-1), "mixed": np.concatenate([recs.reshape(-1)[:500000], gen.text(5, 600000)])}
    seen_filter = False
    for name, a in files.items():
        path = str(d / (name + ".flt"))
        a.tofile(path)
        for opts in (["-cp"], ["-ca"], ["-r"], ["-r", "-ca", "-s"], ["-r", "-cp", "-l"]):
            arch, back = str(d / "f.bsc"), str(d / "f.back")
            _run(REFCLI, "e", path, arch, "-b1", "-t", *([] if "-l" in opts else ["-p"]), *[o for o in opts if o != "-l"])
            raw = open(arch, "rb").read()
            n_blocks = int.from_bytes(raw[4:8], "little")
            seen_filter |= n_blocks > 0 and (raw[8 + 8] > 1 or raw[8 + 9] == 2)    # first record: recordSize, sortingContexts
            _run(TESTCLI, "d", arch, back, "-j3")
            assert open(back, "rb").read() == open(path, "rb").read(), (name, opts)
    assert seen_filter


@pytest.mark.gpu
def test_product_cli_round_trip_on_gpu(gen, tmp_path):
    path, arch, back = str(tmp_path / "in.bin"), str(tmp_path / "a.bsc"), str(tmp_path / "back.bin")
    ri.cli_input(gen).tofile(path)
    _run(PRODUCT, "e", path, arch, *ri.CLI_OPTS, "-j5")
    _run(PRODUCT, "d", arch, back, "-j5")
    assert open(back, "rb").read() == open(path, "rb").read()
    ours = open(arch, "rb").read()
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_results.json")))["cli_archive"]   # `bsc e in out -b8 -p -t`
    assert {"size": len(ours), "sha256": hashlib.sha256(ours).hexdigest()} == gold


@pytest.mark.gpu
def test_reference_cli_with_our_stage_library_on_gpu(gen, tmp_path):
    """INTEGRATION.md option 1, executed: oracle/_ref/bsc_dropin = the reference's own bsc.cpp + libbsc.cpp + host stages linked against
    libbsc_b200.so for the stage entry points.  Its archives must equal the stock reference binary's, each must decode the other's, for
    BWT and ST blocks, with the reference's default LZP stage on and off."""
    dropin = os.path.join(REFDIR, "bsc_dropin")
    if not (os.path.exists(dropin) and os.path.exists(REFCLI)):
        pytest.skip("oracle/_ref/bsc_dropin not built (needs /root/reference at build time)")
    path = str(tmp_path / "in.bin")
    np.concatenate([gen.text(2, 5 << 20), np.tile(gen.text(3, 700), 900), gen.skew(3, 1 << 20)]).tofile(path)
    for opts in (["-b2", "-p"], ["-b2"], ["-b3", "-m5", "-p"], ["-b2", "-e2", "-p"]):
        ours, theirs, back = str(tmp_path / "o.bsc"), str(tmp_path / "t.bsc"), str(tmp_path / "b.bin")
        _run(dropin, "e", path, ours, *opts, "-t")
        _run(REFCLI, "e", path, theirs, *opts, "-t")
        assert open(ours, "rb").read() == open(theirs, "rb").read(), opts
        _run(dropin, "d", theirs, back)
        assert open(back, "rb").read() == open(path, "rb").read(), opts
        _run(REFCLI, "d", ours, back)
        assert open(back, "rb").read() == open(path, "rb").read(), opts
