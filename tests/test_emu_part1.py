"""CPU-only: the kernels that serve combined herumi-API calls, run on the host (tests/emu/emu_part1.cpp).  k_single over a mix of n
ops in one launch (thread i = op i) gives the results of the same ops launched one at a time, and those equal the oracle's; the
index form of k_broadcast_hm gathers H(m) table entries to requests, the null-index form still broadcasts entry 0."""
import ctypes, os, subprocess
import pytest
from harmony_b200 import workload as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OP_G1_ADD, OP_G1_SUB, OP_G2_ADD, OP_G1_EQ, OP_G2_EQ, OP_G1_SER, OP_G2_SER, OP_G1_DES, OP_G2_DES, OP_MAP_SER = range(1, 11)

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "emu", "emu_part1.cpp")
    out = str(tmp_path_factory.mktemp("emu") / "libhbls_emu_part1.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out, src])
    L = ctypes.CDLL(out)
    L.emu_single_mix.argtypes = [ctypes.c_size_t, ctypes.POINTER(ctypes.c_int), ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(ctypes.c_int)]
    L.emu_hm_gather.argtypes = [ctypes.c_size_t, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint32)]
    return L

def mix(emu, slots, ops):
    """ops: (op, slot a, slot b, len); returns per-op (rc, 288 output bytes) of the combined launch (asserted equal to lone launches)."""
    n = len(ops)
    flat = (ctypes.c_int * (4 * n))(*[v for o in ops for v in o])
    blob = b"".join(s.ljust(288, b"\0") for s in slots)
    out = ctypes.create_string_buffer(288 * n); rc = (ctypes.c_int * n)()
    r = emu.emu_single_mix(n, flat, blob, out, rc)
    assert r == 0, f"op {r - 1} differs between the combined launch and a lone launch"
    return [(rc[i], out.raw[288 * i:288 * i + 288]) for i in range(n)]

def test_single_ops_combined_equal_lone(emu, oracle):
    sks = [wl.sk_bytes(wl.seeded_sk("emu-p1", i)) for i in range(2)]
    pks = [oracle.get_public_key(k) for k in sks]
    m = [wl.seeded_bytes("emu-p1/m", i, 32) for i in range(2)]
    sigs = [oracle.sign_hash(k, x) for k, x in zip(sks, m)]
    # Deserialize: valid and undecodable keys / signatures in one launch
    r = mix(emu, [pks[0], pks[1], b"\xff" * 48, sigs[0], sigs[1], b"\xff" * 96],
            [(OP_G1_DES, 0, -1, 0), (OP_G1_DES, 1, -1, 0), (OP_G1_DES, 2, -1, 0), (OP_G2_DES, 3, -1, 0), (OP_G2_DES, 4, -1, 0), (OP_G2_DES, 5, -1, 0)])
    assert [x[0] for x in r] == [48, 48, 0, 96, 96, 0]
    P0, P1, S0, S1 = r[0][1][:144], r[1][1][:144], r[3][1], r[4][1]
    msg = wl.seeded_bytes("emu-p1/map", 0, 32)
    # Add / Sub / SignatureAdd / IsEqual / Serialize / hbls_map_to_g2 (valid and undefined) in one launch
    r = mix(emu, [P0, P1, S0, S1, msg, bytes(32)],
            [(OP_G1_ADD, 0, 1, 0), (OP_G1_SUB, 0, 1, 0), (OP_G2_ADD, 2, 3, 0), (OP_G1_EQ, 0, 0, 0), (OP_G1_EQ, 0, 1, 0),
             (OP_G2_EQ, 2, 2, 0), (OP_G2_EQ, 2, 3, 0), (OP_G1_SER, 0, -1, 0), (OP_G2_SER, 3, -1, 0), (OP_MAP_SER, 4, -1, 32), (OP_MAP_SER, 5, -1, 32)])
    assert [x[0] for x in r] == [0, 0, 0, 1, 0, 1, 0, 48, 96, 0, -1]
    assert r[7][1][:48] == pks[0] and r[8][1][:96] == sigs[1]
    assert r[9][1][:96] == oracle.map_to_g2(msg)
    # the sums, serialized in a third launch
    r = mix(emu, [r[0][1][:144], r[1][1][:144], r[2][1]], [(OP_G1_SER, 0, -1, 0), (OP_G1_SER, 1, -1, 0), (OP_G2_SER, 2, -1, 0)])
    assert r[0][1][:48] == oracle.pk_add(pks[0], pks[1])
    assert r[1][1][:48] == oracle.pk_add(pks[0], pks[1], sub=True)
    assert r[2][1][:96] == oracle.sig_add(sigs[0], sigs[1])

def test_hm_index_gather(emu):
    for n, nsrc, idx in ((5, 3, [2, 0, 0, 1, 2]), (1, 1, [0]), (300, 7, [(i * 5) % 7 for i in range(300)])):
        assert emu.emu_hm_gather(n, nsrc, (ctypes.c_uint32 * n)(*idx)) == 0, (n, nsrc)
