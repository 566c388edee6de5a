"""CPU-only: the message-grouping and status kernels of harmony_b200/csrc/device_forms.cuh run on the host
(tests/emu/emu_device_forms.cpp).  Grouping: items whose messages agree in the 48 zero-padded bytes the map reads are one message,
represented by their lowest index, numbered in item order, whatever order the "threads" run in.  Statuses: the status kernels are
the only library code that assigns HBLS_VB_* / HBLS_HDR_*, for the host and the device forms alike; the order of checks (key, then signature
encoding, then VerifyHash; encoding, then quorum, then VerifyHash) is restated independently here and checked on every combination
of the k_pack_flags bits."""
import ctypes, itertools, os, random, subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(ROOT, "tests", "emu", "emu_device_forms.cpp")
    out = os.path.join(ROOT, "tests", "emu", "libhbls_emu_device_forms.so")
    csrc = os.path.join(ROOT, "harmony_b200", "csrc")
    deps = [src, os.path.join(ROOT, "include", "hbls.h")] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out, src])
    L = ctypes.CDLL(out)
    c = ctypes
    L.emu_group.argtypes = [c.c_size_t, c.c_char_p, c.c_uint32, c.c_int, c.c_uint64, c.c_uint64, c.POINTER(c.c_uint), c.c_void_p, c.c_void_p, c.c_void_p]
    L.emu_group_hash.argtypes = [c.c_char_p, c.c_uint32, c.c_size_t, c.c_uint64, c.c_uint64]
    L.emu_group_hash.restype = c.c_uint64
    L.emu_status_triples.argtypes = [c.c_size_t, c.c_char_p, c.c_char_p, c.c_void_p]
    L.emu_status_headers.argtypes = [c.c_size_t, c.c_size_t, c.c_char_p, c.c_size_t, c.c_size_t, c.c_char_p, c.c_char_p, c.c_void_p]
    return L


def _key(m):
    return (bytes(m[:48]) + bytes(48))[:48]


def group(emu, msgs, msg_len, reverse=0, key=(0x0706050403020100, 0x0f0e0d0c0b0a0908)):
    k = len(msgs)
    blob = b"".join(msgs)
    assert len(blob) == k * msg_len
    d = ctypes.c_uint(0xdead)
    grp = (ctypes.c_uint32 * k)(); rep = (ctypes.c_uint32 * k)(); keys = ctypes.create_string_buffer(48 * k)
    emu.emu_group(k, blob, msg_len, reverse, key[0], key[1], ctypes.byref(d), grp, keys, rep)
    return d.value, list(grp), [keys.raw[48 * i:48 * i + 48] for i in range(d.value)], list(rep)


def expected(msgs):
    first, order, grp, rep = {}, [], [], []
    for i, m in enumerate(msgs):
        key = _key(m)
        if key not in first:
            first[key] = i; order.append(key)
        grp.append(order.index(key)); rep.append(first[key])
    return len(order), grp, order, rep


def check(emu, msgs, msg_len):
    want = expected(msgs)
    for reverse in (0, 1):
        for key in ((0x0706050403020100, 0x0f0e0d0c0b0a0908), (0xdeadbeef12345678, 0x1)):      # the table key moves slots, not results
            assert group(emu, msgs, msg_len, reverse, key) == want, (reverse, key)
    return want


def test_first_48_bytes_decide(emu):
    base = bytes(range(1, 49))
    msgs = [base + bytes([i]) * 16 for i in range(6)] + [bytes([9]) + base[1:] + bytes(16)]
    d, grp, keys, rep = check(emu, msgs, 64)
    assert d == 2 and grp == [0] * 6 + [1] and keys[0] == base and rep == [0] * 6 + [6]


def test_short_messages_zero_padded(emu):
    msgs = [b"\x01" * 20, b"\x01" * 19 + b"\x00", b"\x01" * 20, b"\x02" * 20]
    d, grp, keys, _ = check(emu, msgs, 20)
    assert d == 3 and grp == [0, 1, 0, 2] and keys[0] == b"\x01" * 20 + bytes(28)


def test_zero_length_and_t0_message(emu):
    assert check(emu, [b""] * 5, 0)[:2] == (1, [0] * 5)
    d, grp, keys, _ = check(emu, [bytes(32), b"\x05" * 32, bytes(32)], 32)      # the t = 0 message is a message like any other
    assert d == 2 and grp == [0, 1, 0] and keys[0] == bytes(48)


def test_all_distinct_all_equal_single(emu):
    distinct = [i.to_bytes(4, "little") * 12 for i in range(200)]
    assert check(emu, distinct, 48)[:2] == (200, list(range(200)))
    assert check(emu, [b"\x07" * 48] * 200, 48)[:2] == (1, [0] * 200)
    assert check(emu, [b"\x07" * 40], 40)[:2] == (1, [0])


def test_many_repeats_and_table_collisions(emu):
    rng = random.Random(7)
    pool = [bytes(rng.randrange(256) for _ in range(48)) for _ in range(37)]
    msgs = [rng.choice(pool) for _ in range(500)]                 # the view-change shape: few messages, many items
    d, grp, keys, rep = check(emu, msgs, 48)
    assert d == len(set(msgs)) and all(msgs[rep[i]] == msgs[i] and rep[i] <= i for i in range(500))
    msgs = [bytes(rng.randrange(4) for _ in range(48)) for _ in range(64)]     # a full table of 128 slots: long probe chains
    check(emu, msgs + msgs[::-1], 48)


def _status_triple(f, r):
    return 4 if not f & 4 else 3 if not f & 1 else 1 if r == 1 else 0


def _status_header(f, r, bm, nslots, quorum):
    set_bits = sum(1 for i in range(nslots) if bm[i >> 3] >> (i & 7) & 1)
    return 3 if not f & 1 else 2 if quorum and set_bits < quorum else 1 if r else 0


def test_status_triples_every_flag_combination(emu):
    cases = list(itertools.product(range(8), (0, 1, 2)))
    flags = bytes(f for f, _ in cases); res = bytes(r for _, r in cases)
    out = ctypes.create_string_buffer(len(cases))
    emu.emu_status_triples(len(cases), flags, res, out)
    assert list(out.raw) == [_status_triple(f, r) for f, r in cases]


def test_status_headers_every_flag_combination_and_padding(emu):
    nslots, blen = 13, 2
    bitmaps = [bytes([0xff, 0xff]), bytes([0xff, 0x1f]), bytes([0x00, 0xe0]), bytes([0x0f, 0xe0]), bytes([0x00, 0x00]), bytes([0xfe, 0x1f])]
    for quorum in (0, 1, 4, 5, 12, 13, 14):
        cases = list(itertools.product(range(8), (0, 1, 2), bitmaps))
        out = ctypes.create_string_buffer(len(cases))
        emu.emu_status_headers(len(cases), nslots, b"".join(b for _, _, b in cases), blen, quorum, bytes(f for f, _, _ in cases),
                               bytes(r for _, r, _ in cases), out)
        assert list(out.raw) == [_status_header(f, r, b, nslots, quorum) for f, r, b in cases], quorum


def _siphash24(k0, k1, data):
    """SipHash-2-4 (Aumasson, Bernstein 2012) of data (a multiple of 8 bytes here) under the key (k0, k1)"""
    M = (1 << 64) - 1
    rotl = lambda x, b: ((x << b) | (x >> (64 - b))) & M
    v = [k0 ^ 0x736f6d6570736575, k1 ^ 0x646f72616e646f6d, k0 ^ 0x6c7967656e657261, k1 ^ 0x7465646279746573]
    def rnd():
        v[0] = (v[0] + v[1]) & M; v[1] = rotl(v[1], 13) ^ v[0]; v[0] = rotl(v[0], 32)
        v[2] = (v[2] + v[3]) & M; v[3] = rotl(v[3], 16) ^ v[2]
        v[0] = (v[0] + v[3]) & M; v[3] = rotl(v[3], 21) ^ v[0]
        v[2] = (v[2] + v[1]) & M; v[1] = rotl(v[1], 17) ^ v[2]; v[2] = rotl(v[2], 32)
    for m in [int.from_bytes(data[i:i + 8], "little") for i in range(0, len(data), 8)] + [(len(data) & 0xff) << 56]:
        v[3] ^= m; rnd(); rnd(); v[0] ^= m
    v[2] ^= 0xff
    for _ in range(4): rnd()
    return v[0] ^ v[1] ^ v[2] ^ v[3]


def test_table_hash_is_keyed_siphash(emu):
    """The slot hash is SipHash-2-4 of the 48 zero-padded key bytes under the call's key: a sender who does not know the key cannot
    choose messages that pile up in one probe chain."""
    rng = random.Random(11)
    for msg_len in (48, 64, 20, 0):
        msgs = [bytes(rng.randrange(256) for _ in range(msg_len)) for _ in range(4)]
        for key in ((0x0706050403020100, 0x0f0e0d0c0b0a0908), (rng.getrandbits(64), rng.getrandbits(64))):
            for i, m in enumerate(msgs):
                assert emu.emu_group_hash(b"".join(msgs), msg_len, i, *key) == _siphash24(*key, _key(m))
    key = (0x0706050403020100, 0x0f0e0d0c0b0a0908)
    assert emu.emu_group_hash(bytes(range(48)), 48, 0, *key) != emu.emu_group_hash(bytes(range(48)), 48, 0, key[0] ^ 1, key[1])
