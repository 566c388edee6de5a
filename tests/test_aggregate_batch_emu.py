"""CPU-only: the kernels of hbls_aggregate_sigs_batch (k_g2_segsum_plan, k_g2_segsum_chunks, k_g2_segsum_fold) run on the host
(tests/emu/emu_aggregate_batch.cpp) with the chunk size shrunk to a few rows, so every set spans chunks and every branch runs: chunk
starts and ends inside and at the edges of a set, lanes without rows, the plan's scan over several tiles, a bad range, sets summed by
their fold warp because overlapping ranges overflow the chunk table.  Each set's bytes and status are compared with the CPU oracle's
AggregateSig (ho_aggregate_sigs): its sum when every signature decodes, else the identity's encoding."""
import ctypes, os, random, subprocess, sys, tempfile
import pytest
from harmony_b200 import workload as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import pyref as o                                   # noqa: E402
from gen_selftest import reject_encodings           # noqa: E402

AGG_OK, AGG_BAD_SIG_ENCODING, AGG_BAD_RANGE = 32, 33, 34
_BUILD = tempfile.mkdtemp(prefix="hbls_aggb_")


@pytest.fixture(scope="module", params=[5, 37])
def emu(request):
    """the harness built with HB_AGG_CHUNK = 5 (most lanes idle) and 37 (lanes with two rows)"""
    chunk = request.param
    out = os.path.join(_BUILD, f"libemu_aggb_{chunk}.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", f"-DHB_AGG_CHUNK={chunk}", "-o", out,
                           os.path.join(ROOT, "tests", "emu", "emu_aggregate_batch.cpp")])
    L = ctypes.CDLL(out)
    L.emu_agg_chunk.restype = ctypes.c_uint32
    L.emu_agg_batch.argtypes = [ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint, ctypes.c_char_p,
                                ctypes.c_char_p, ctypes.POINTER(ctypes.c_uint32)]
    assert L.emu_agg_chunk() == chunk
    return L


@pytest.fixture(scope="module")
def pool(oracle):
    """valid signatures, their negations, and the three reject classes (x >= p, off the curve, outside the subgroup)"""
    sigs = [oracle.sign_hash(wl.sk_bytes(wl.seeded_sk("aggb", i)), wl.commit_payload("aggb", i)) for i in range(12)]
    neg = [o.g2_serialize(o.pt_neg(o.FP2, o.g2_deserialize(s))) for s in sigs[:3]]
    _, g2r = reject_encodings()
    return sigs, neg, g2r


def run(emu, offsets, rows, plan_threads=4):
    B, n = len(offsets) - 1, len(rows)
    off = (ctypes.c_uint64 * (B + 1))(*offsets)
    out = ctypes.create_string_buffer(96 * B); st = ctypes.create_string_buffer(B); direct = ctypes.c_uint32(0)
    emu.emu_agg_batch(B, n, off, b"".join(rows) or b"\x00", plan_threads, out, st, ctypes.byref(direct))
    return [out.raw[96 * j:96 * j + 96] for j in range(B)], list(st.raw[:B]), direct.value


def expected(oracle, offsets, rows):
    ident = oracle.aggregate_sigs([])
    outs, sts = [], []
    for j in range(len(offsets) - 1):
        lo, hi = offsets[j], offsets[j + 1]
        if lo > hi or hi > len(rows): outs.append(ident); sts.append(AGG_BAD_RANGE); continue
        agg = oracle.aggregate_sigs(rows[lo:hi])
        outs.append(agg if agg is not None else ident); sts.append(AGG_OK if agg is not None else AGG_BAD_SIG_ENCODING)
    return outs, sts


def check(emu, oracle, offsets, rows, plan_threads=4):
    got_out, got_st, direct = run(emu, offsets, rows, plan_threads)
    exp_out, exp_st = expected(oracle, offsets, rows)
    assert got_st == exp_st
    assert got_out == exp_out
    return got_st, direct


def sizes_to_offsets(sizes):
    off = [0]
    for s in sizes: off.append(off[-1] + s)
    return off


def test_set_sizes_around_the_chunk(emu, oracle, pool):
    """empty sets, sets of C - 1, C, C + 1 and several C rows, one row, back to back"""
    sigs, _, _ = pool
    C = emu.emu_agg_chunk()
    rng = random.Random(C)
    sizes = [0, 1, C - 1, C, C + 1, 0, 2 * C, 3 * C + 2, 0] if C < 10 else [0, 1, C - 1, C, C + 1, 0, 2 * C + 3]
    rows = [rng.choice(sigs) for _ in range(sum(sizes))]
    st, direct = check(emu, oracle, sizes_to_offsets(sizes), rows)
    assert st == [AGG_OK] * len(sizes) and direct == 0


def test_plan_scan_over_tiles(emu, oracle, pool):
    """B larger than the plan CTA: the exclusive scan carries over tiles, for CTAs of 1, 3 and 4 threads"""
    sigs, _, _ = pool
    C = emu.emu_agg_chunk()
    rng = random.Random(7)
    sizes = [rng.choice([0, 1, 2, C, C + 1]) for _ in range(11)]
    rows = [rng.choice(sigs) for _ in range(sum(sizes))]
    for t in (1, 3, 4):
        check(emu, oracle, sizes_to_offsets(sizes), rows, t)


def test_bad_signatures_at_chunk_starts_ends_and_middle(emu, oracle, pool):
    """each reject class at the first, last and a middle row of a chunk, and at the last row of a set; the other sets stay exact"""
    sigs, _, g2r = pool
    C = emu.emu_agg_chunk()
    rng = random.Random(11)
    places = [0, C - 1, C // 2, C, 2 * C - 1]
    for k, bad in enumerate(g2r):
        for p in places:
            size = 2 * C + 1
            rows = [rng.choice(sigs) for _ in range(3 * size)]
            rows[size + p] = bad                               # middle set: bad row at position p
            st, _ = check(emu, oracle, [0, size, 2 * size, 3 * size], rows)
            assert st == [AGG_OK, AGG_BAD_SIG_ENCODING, AGG_OK], (k, p)
    rows = [rng.choice(sigs) for _ in range(C + 2)]; rows[-1] = g2r[2]
    assert check(emu, oracle, [0, 1, C + 2], rows)[0] == [AGG_OK, AGG_BAD_SIG_ENCODING]


def test_identity_sums(emu, oracle, pool):
    """sigma + (-sigma) in one chunk and across chunks, and a set of identity encodings: the identity, status OK"""
    sigs, neg, _ = pool
    C = emu.emu_agg_chunk()
    ident = oracle.aggregate_sigs([])
    fill = [sigs[3 + i % 6] for i in range(C)]
    sets = [[sigs[0], neg[0]], [neg[1], sigs[1]], [sigs[2]] + [ident] * C + [neg[2]], [ident] * 3]
    across = [sigs[0]] + fill[:C - 1] + [neg[0]] + [neg[0]] + fill[:C - 1] + [sigs[0]]      # sigma at a chunk start, -sigma in the next chunk
    sets.append(across)
    rows = [r for s in sets for r in s]
    out, st, _ = run(emu, sizes_to_offsets([len(s) for s in sets]), rows)
    assert st == [AGG_OK] * len(sets)
    assert out[:4] == [ident] * 4
    assert out[4] == oracle.aggregate_sigs(fill[:C - 1] * 2) == expected(oracle, [0, len(across)], across)[0][0]


def test_bad_ranges(emu, oracle, pool):
    """decreasing offsets and offsets past n give BAD_RANGE and the identity; a set starting at the last row; offsets[0] need not be 0"""
    sigs, _, _ = pool
    C = emu.emu_agg_chunk()
    n = 3 * C + 2
    rows = [sigs[i % len(sigs)] for i in range(n)]
    st, _ = check(emu, oracle, [0, C, 2, C + 3, n - 1, n, n + 1, n + 1, n, n], rows)
    assert st == [AGG_OK, AGG_BAD_RANGE, AGG_OK, AGG_OK, AGG_OK, AGG_BAD_RANGE, AGG_BAD_RANGE, AGG_BAD_RANGE, AGG_OK]
    st, _ = check(emu, oracle, [C, n, 1 << 63, 0, n - 1], rows)
    assert st == [AGG_OK, AGG_BAD_RANGE, AGG_BAD_RANGE, AGG_OK]


def test_overlapping_sets_overflow_the_chunk_table(emu, oracle, pool):
    """valid sets that overlap through reversed ones in between need more chunks than ceil(n / C) + B: the sets past the table are
    summed by their fold warp, with the same bytes"""
    sigs, _, g2r = pool
    C = emu.emu_agg_chunk()
    n = 4 * C
    rows = [sigs[i % len(sigs)] for i in range(n)]
    rows[C + 1] = g2r[0]
    offsets = [0]
    for _ in range(4): offsets += [n, 0]                       # [0, n) valid, [n, 0) reversed, ...
    offsets += [C + 2]
    st, direct = check(emu, oracle, offsets, rows)
    assert st == [AGG_BAD_SIG_ENCODING, AGG_BAD_RANGE] * 4 + [AGG_BAD_SIG_ENCODING]
    assert direct > 0
    offsets = [0] + [n, C + 2] * 5 + [n]                     # [C + 2, n): every row decodes
    st, direct = check(emu, oracle, offsets, rows)
    assert st == [AGG_BAD_SIG_ENCODING] + [AGG_BAD_RANGE, AGG_OK] * 5 and direct > 0


def test_no_rows(emu, oracle):
    out, st, _ = run(emu, [0, 0, 0], [])
    assert st == [AGG_OK, AGG_OK] and out == [oracle.aggregate_sigs([])] * 2
