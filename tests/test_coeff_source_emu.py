"""CPU-only: the secrets of device-form calls captured into a CUDA graph, on the host (tests/emu/emu_coeff_source.cpp).

Captured calls draw their random-linear-combination coefficients and message-grouping salt on the device, at every replay
(kernels.cuh k_rlc_draw), and the kernels read them through device pointers.  Here: the device ChaCha20 block function returns the
block of RFC 8439 section 2.3.2 and agrees with the host stream's block function (chacha20.hpp) for random keys, counters and block
numbers; the device stream's nonce word is not the host stream's; and every scaling kernel hbls.cu launches, and k_group_insert, give
the same bytes (points, bad flags, slots) whether their coefficients / salt come by value or through the pointer sources."""
import ctypes, os, random, subprocess, tempfile
import pytest
from harmony_b200 import workload as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_BUILD = tempfile.mkdtemp(prefix="hbls_coeff_source_")
_NCO = 8 + 8 * 16
_HOST_NONCE = 0x68626c73


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(ROOT, "tests", "emu", "emu_coeff_source.cpp")
    out = os.path.join(_BUILD, "libemu_coeff_source.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out, src])
    L = ctypes.CDLL(out)
    c = ctypes
    L.emu_chacha_dev.argtypes = [c.POINTER(c.c_uint32), c.POINTER(c.c_uint32)]
    L.emu_chacha_host.argtypes = [c.POINTER(c.c_uint32), c.c_uint64, c.c_uint32, c.POINTER(c.c_uint32)]
    L.emu_draw_nonce.restype = c.c_uint32
    L.emu_scale_sources.argtypes = [c.c_int, c.c_size_t, c.c_char_p, c.c_char_p, c.c_char_p, c.c_uint32, c.c_size_t, c.POINTER(c.c_uint64), c.c_int, c.c_int]
    L.emu_group_sources.argtypes = [c.c_size_t, c.c_char_p, c.c_uint32, c.c_uint64, c.c_uint64, c.c_uint64, c.c_uint64]
    return L


def _dev_block(emu, state):
    st = (ctypes.c_uint32 * 16)(*state); out = (ctypes.c_uint32 * 16)()
    emu.emu_chacha_dev(st, out)
    return list(out)


def test_rfc8439_block_vector(emu):
    key = [int.from_bytes(bytes(range(4 * i, 4 * i + 4)), "little") for i in range(8)]
    state = [0x61707865, 0x3320646e, 0x79622d32, 0x6b206574] + key + [0x00000001, 0x09000000, 0x4a000000, 0x00000000]
    assert _dev_block(emu, state) == [0xe4e7f110, 0x15593bd1, 0x1fdd0f50, 0xc47120a3, 0xc7f4d1c7, 0x0368c033, 0x9aaa2204, 0x4e6cd4c3,
                                      0x466482d2, 0x09aa9f07, 0x05d7c214, 0xa2028bd9, 0xd19c12b5, 0xb94e16de, 0xe883d0cb, 0x4e3c50a2]


def test_device_block_matches_host_stream(emu):
    rng = random.Random(8439)
    for t in range(200):
        key = [rng.getrandbits(32) for _ in range(8)]
        counter = rng.choice([0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 64 - 1, rng.getrandbits(64)])
        block = rng.choice([0, 1, 17, 2 ** 32 - 1, rng.getrandbits(32)])
        want = (ctypes.c_uint32 * 16)()
        emu.emu_chacha_host((ctypes.c_uint32 * 8)(*key), counter, block, want)
        state = [0x61707865, 0x3320646e, 0x79622d32, 0x6b206574] + key + [counter & 0xffffffff, counter >> 32, _HOST_NONCE, block]
        assert _dev_block(emu, state) == list(want), t


def test_device_draws_use_their_own_nonce(emu):
    assert emu.emu_draw_nonce() != _HOST_NONCE


def _rounds(oracle, n, seed):
    """n rounds with undecodable and identity signatures, identity keys and an undefined map at seeded positions"""
    rng = random.Random(seed)
    sks = [wl.seeded_sk("cs-emu", i) for i in range(8)]
    pks = [oracle.get_public_key(wl.sk_bytes(k)) for k in sks]
    keys, sigs, msgs = [], [], []
    for j in range(n):
        k = rng.randrange(8); m = wl.commit_payload("cs-emu%d" % seed, j); c = rng.randrange(10)
        if c == 3: m = bytes(48)
        s = oracle.sign_hash(wl.sk_bytes(sks[k]), m if c != 3 else b"y" * 48)
        if c == 0: s = b"\xff" * 96
        elif c == 1: s = bytes(96)
        elif c == 4: s = sigs[-1] if sigs else s
        keys.append(bytes(48) if c == 2 else pks[k]); sigs.append(s); msgs.append(m)
    return b"".join(keys), b"".join(sigs), b"".join(msgs)


@pytest.mark.parametrize("G,ng,blocks,gate", [(4, 3, 0, -1), (4, 3, 1, -1), (8, 2, 1, 1), (8, 2, 1, 0), (4, 2, 0, 0)])
def test_scaling_kernels_same_bytes_from_either_source(emu, oracle, G, ng, blocks, gate):
    n = G * ng
    keys, sigs, msgs = _rounds(oracle, n, G * 100 + ng * 10 + blocks * 2 + gate)
    rng = random.Random(n + blocks + gate)
    co = (ctypes.c_uint64 * _NCO)(*[rng.getrandbits(64) for _ in range(_NCO)])
    assert emu.emu_scale_sources(G, n, keys, sigs, msgs, 48, ng, co, blocks, gate) == 0


def test_group_insert_same_slots_from_either_source(emu):
    rng = random.Random(52)
    for k, msg_len in ((1, 32), (40, 32), (97, 48), (130, 64)):
        pool = [wl.seeded_bytes("cs-grp", i, msg_len) for i in range(max(1, k // 3))]
        msgs = b"".join(pool[rng.randrange(len(pool))] for _ in range(k))
        k0, k1 = rng.getrandbits(64), rng.getrandbits(64)
        assert emu.emu_group_sources(k, msgs, msg_len, k0, k1, k0, k1) == 0, k
    # the pointer really is read: another salt moves the slots of a large enough table
    msgs = b"".join(wl.seeded_bytes("cs-grp2", i, 32) for i in range(64))
    assert emu.emu_group_sources(64, msgs, 32, 1, 2, 3, 4) > 0
