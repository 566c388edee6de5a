"""CPU-only: the descriptor kernels of the committee-set form (hbls_aggregate_verify_set_device: k_set_tile_sums, k_set_tile_scan,
k_set_items, k_set_bad_index in harmony_b200/csrc/kernels.cuh) run on the host (tests/emu/emu_committee_set.cpp) with the scan tile
shrunk to a few items, so that every batch spans several tiles and the tile scan carries over several passes of its CTA.  For the
items with a valid index the descriptors must be exactly what the host-array form builds (hbls.cu verify_items_body: each item's
committee, its slots, and its bitmap at the running sum of the bitmap bytes of the items before it); an item with a bad index names
no committee, has no bitmap and no slots, takes no bitmap bytes, and ends as HBLS_SET_BAD_INDEX whatever verdict the tail wrote.
Also: the new entry points are exported, and the new kernels compile for sm_90a without local-memory spills."""
import ctypes, os, random, re, subprocess, tempfile
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SET_BAD_INDEX = 48
_BUILD = tempfile.mkdtemp(prefix="hbls_set_")
BAD = 0xffffffff


@pytest.fixture(scope="module", params=[4, 7])
def emu(request):
    """the harness built with HB_SET_TILE = 4 and 7 (a power of two and not)"""
    tile = request.param
    out = os.path.join(_BUILD, f"libemu_set_{tile}.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", f"-DHB_SET_TILE={tile}", "-o", out,
                           os.path.join(ROOT, "tests", "emu", "emu_committee_set.cpp")])
    L = ctypes.CDLL(out)
    L.emu_set_tile.restype = ctypes.c_uint32
    L.emu_set_items.argtypes = [ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_uint, ctypes.c_void_p,
                                ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    assert L.emu_set_tile() == tile
    return L


def run(emu, index, slots, scan_threads=None, verdicts=None):
    k, m = len(index), len(slots)
    scan_threads = scan_threads or emu.emu_set_tile()
    idx = (ctypes.c_uint32 * max(k, 1))(*index); sl = (ctypes.c_uint64 * m)(*slots)
    com = (ctypes.c_int64 * max(k, 1))(); off = (ctypes.c_uint64 * max(k, 1))(); n = (ctypes.c_uint64 * max(k, 1))()
    ok = ctypes.create_string_buffer(max(k, 1))
    res = ctypes.create_string_buffer(bytes(verdicts) if verdicts is not None else bytes(j % 2 for j in range(k)) or b"\x00")
    emu.emu_set_items(k, idx, m, sl, scan_threads, com, off, n, ok, res)
    return [(com[j], off[j], n[j], ok.raw[j]) for j in range(k)], res.raw[:k]


def host_array_descriptors(committees_slots):
    """hbls.cu verify_items_body, restated: (slots, bitmap offset) per item of a host array of committees"""
    out, off = [], 0
    for n in committees_slots:
        out.append((n, off)); off += (n + 7) >> 3
    return out


def check(emu, index, slots, scan_threads=None):
    got, res = run(emu, index, slots, scan_threads)
    m = len(slots)
    valid = [j for j, i in enumerate(index) if i < m]
    want = host_array_descriptors([slots[index[j]] for j in valid])
    assert [(got[j][2], got[j][1]) for j in valid] == want
    assert [got[j][0] for j in valid] == [index[j] for j in valid] and all(got[j][3] == 1 for j in valid)
    for j, i in enumerate(index):
        if i >= m:
            assert got[j] == (-1, 2 ** 64 - 1, 0, 0), j
    verdicts = bytes(j % 2 for j in range(len(index)))
    assert res == bytes(SET_BAD_INDEX if i >= m else verdicts[j] for j, i in enumerate(index))
    return got


SIZES = [1, 7, 8, 9, 250, 1000]


def test_every_committee_size_across_tiles(emu):
    """committees of 1, 7, 8, 9, 250 and 1 000 slots, items in a seeded order over many tiles"""
    rng = random.Random(3)
    index = [rng.randrange(len(SIZES)) for _ in range(61)]
    check(emu, index, SIZES)
    check(emu, list(range(len(SIZES))) * 5, SIZES)


def test_offsets_at_tile_boundaries(emu):
    """batches of T - 1, T, T + 1, 2T and 3T + 1 items: the first and last item of every tile carry the right offset"""
    T = emu.emu_set_tile()
    for k in (1, T - 1, T, T + 1, 2 * T, 3 * T + 1):
        index = [j % len(SIZES) for j in range(k)]
        got = check(emu, index, SIZES)
        assert got[-1][1] == sum((SIZES[i] + 7) >> 3 for i in index[:-1])


def test_tile_scan_over_several_passes(emu):
    """more tiles than the tile-scan CTA has threads: its scan carries over passes, for CTAs of 1, 2, 3 and T threads"""
    T = emu.emu_set_tile()
    rng = random.Random(5)
    index = [rng.randrange(len(SIZES)) for _ in range(9 * T + 2)]
    for t in sorted({1, 2, 3, T}):
        check(emu, index, SIZES, t)


def test_bad_indices_first_last_middle(emu):
    """an index equal to m, and 2^32 - 1 (a negative int32), at the first, a middle and the last position, alone and in runs; the
    other items keep the offsets of the batch without them"""
    T = emu.emu_set_tile()
    rng = random.Random(9)
    base = [rng.randrange(len(SIZES)) for _ in range(4 * T + 3)]
    m = len(SIZES)
    for bad in (m, BAD, m + 1000):
        for places in ([0], [len(base) // 2], [len(base) - 1], [0, len(base) // 2, len(base) - 1], [T - 1, T, T + 1]):
            index = list(base)
            for p in places: index[p] = bad
            check(emu, index, SIZES)


def test_all_bad_and_single_item(emu):
    got = check(emu, [BAD] * 10, SIZES)
    assert all(g == (-1, 2 ** 64 - 1, 0, 0) for g in got)
    assert check(emu, [3], SIZES) == [(3, 0, 9, 1)]
    assert check(emu, [len(SIZES)], SIZES) == [(-1, 2 ** 64 - 1, 0, 0)]


def test_one_committee_set(emu):
    """a set of one committee (m = 1): index 1 is already bad"""
    check(emu, [0, 1, 0, 0, 1, 1, 0] * 3, [250])


def test_bad_index_overrides_every_verdict(emu):
    """k_set_bad_index writes HBLS_SET_BAD_INDEX over 0, 1 and any other byte the tail left, and nothing else"""
    index = [0, BAD, 1, BAD, 2, BAD]
    for verdicts in (bytes(6), b"\x01" * 6, bytes([0xee, 1, 0, 3, 1, 0])):
        _, res = run(emu, index, [8, 9, 250], None, verdicts)
        assert res == bytes([verdicts[0], SET_BAD_INDEX, verdicts[2], SET_BAD_INDEX, verdicts[4], SET_BAD_INDEX])


# ---------------------------------------------------------------------------------------------------------------- ABI and build
def test_committee_set_symbols_exported():
    from harmony_b200 import build
    L = ctypes.CDLL(build.build_cuda())
    for name in ("hbls_committee_set_create", "hbls_committee_set_destroy", "hbls_committee_set_size", "hbls_aggregate_verify_set_device"):
        assert hasattr(L, name), name
    hdr = open(os.path.join(ROOT, "include", "hbls.h")).read()
    assert re.search(r"#define HBLS_SET_BAD_INDEX 48\b", hdr)
    codes = {int(v) for v in re.findall(r"#define HBLS_(?:VB|HDR|BALLOT|AGG)_\w+\s+(\d+)", hdr)}
    assert SET_BAD_INDEX not in codes and {0, 1, 16, 32} <= codes


def test_no_gpu_argument_errors():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from harmony_b200 import bls
    L = bls.lib()
    out = ctypes.c_void_p()
    assert L.hbls_committee_set_create(ctypes.byref(out), None, 0) == bls.ERR_CUDA        # no device: every entry point refuses
    assert L.hbls_aggregate_verify_set_device(None, 0, None, None, None, None, 0, None, None) == bls.ERR_CUDA
    assert L.hbls_committee_set_size(None) == 0


def test_new_kernels_do_not_spill():
    """the sm_90a code of the committee-set kernels in libhbls.so uses no stack and no local memory (no spills)"""
    from harmony_b200 import build
    path = build.build_cuda()
    tool = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("no cuobjdump")
    r = subprocess.run([tool, "--dump-resource-usage", path], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    names = ["k_set_tile_sums", "k_set_tile_scan", "k_set_items", "k_set_bad_index"]
    seen = {}
    for fn, usage in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", r.stdout):
        for n in names:
            if re.search(r"\d" + n + r"E?", fn) or n in fn:
                seen[n] = usage
    assert sorted(seen) == sorted(names), r.stdout[:2000]
    for n, usage in seen.items():
        assert re.search(r"\bSTACK:0\b", usage) and re.search(r"\bLOCAL:0\b", usage), (n, usage)
