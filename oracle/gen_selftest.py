"""
oracle/gen_selftest.py -- known answers of the library's built-in self-test (hbls_self_test).

Writes harmony_b200/csrc/selftest_kat.h: plain C arrays of input bytes and the outputs the C oracle
(oracle/hbls_oracle.c, built by harmony_b200/build.py:build_oracle) gives for them.  Inputs come from fixed seeds
(harmony_b200/workload.py, tag "selftest"); the reject encodings are found by a deterministic search with the
big-integer restatement oracle/pyref.py.  The product includes the header as data and never runs the oracle.
Run:  python oracle/gen_selftest.py        (--check: exit 1 if the committed header differs)
"""
import ctypes, os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import pyref as o                                   # noqa: E402
from harmony_b200 import workload as wl             # noqa: E402

OUT = os.path.join(ROOT, "harmony_b200", "csrc", "selftest_kat.h")
TAG = "selftest"
N_KEYS = 16
MSG_LENS = [1, 8, 32, 40, 48, 64]
N_ROUNDS = 35                 # 4 strided groups of 8 / 8 groups of 4, 3 tail rounds
QUORUM = 2 * N_KEYS // 3 + 1


class Oracle:
    def __init__(self):
        from harmony_b200 import build
        self.L = ctypes.CDLL(build.build_oracle())
    def _out(self, n): return ctypes.create_string_buffer(n)
    def pk(self, sk):
        b = self._out(48); assert self.L.ho_get_public_key(sk, b) == 0; return b.raw
    def sign(self, sk, m):
        b = self._out(96); return b.raw if self.L.ho_sign_hash(sk, m, ctypes.c_size_t(len(m)), b) == 0 else None
    def map(self, m):
        b = self._out(96); return b.raw if self.L.ho_map_to_g2(m, ctypes.c_size_t(len(m)), b) == 0 else None
    def verify(self, sig, pk, m): return self.L.ho_verify_hash(sig, pk, m, ctypes.c_size_t(len(m))) == 1
    def pk_ok(self, pk): return self.L.ho_pk_deserialize_check(pk) == 1
    def sig_ok(self, sig): return self.L.ho_sig_deserialize_check(sig) == 1
    def fp_mul(self, a, b):
        r = self._out(48); assert self.L.ho_fp_mul(a, b, r) == 0; return r.raw
    def pk_add(self, a, b, sub):
        r = self._out(48); assert self.L.ho_pk_add(a, b, sub, r) == 0; return r.raw
    def sig_add(self, a, b):
        r = self._out(96); assert self.L.ho_sig_add(a, b, r) == 0; return r.raw
    def agg_sigs(self, sigs):
        r = self._out(96); assert self.L.ho_aggregate_sigs(ctypes.c_size_t(len(sigs)), b"".join(sigs), r) == 0; return r.raw
    def mask_agg(self, pks, bm):
        r = self._out(48); assert self.L.ho_mask_aggregate(ctypes.c_size_t(len(pks)), b"".join(pks), bm, ctypes.c_size_t(len(bm)), r) == 0
        return r.raw
    def agg_verify(self, pks, bm, sig, m):
        return self.L.ho_fast_aggregate_verify(ctypes.c_size_t(len(pks)), b"".join(pks), bm, ctypes.c_size_t(len(bm)), sig, m, ctypes.c_size_t(len(m))) == 1


def reject_encodings():
    """x >= p, x not on the curve, a curve point outside the order-r subgroup: for G1 (48 B) and G2 (96 B)."""
    P = o.P
    g1 = [P.to_bytes(48, "little")]
    x = 1
    while o.fp_sqrt((x * x * x + o.B1) % P) is not None: x += 1
    g1.append(x.to_bytes(48, "little"))
    x = 1
    while True:
        b = x.to_bytes(48, "little")
        if o.g1_deserialize(b, False) is not None and o.g1_deserialize(b, True) is None: break
        x += 1
    g1.append(b)
    g2 = [P.to_bytes(48, "little") + bytes(48)]
    def on_curve(x2): return o.f2_sqrt(o.f2_add(o.f2_mul(o.f2_sqr(x2), x2), o.B2)) is not None
    t = 1
    while on_curve((t, 0)): t += 1
    g2.append(t.to_bytes(48, "little") + bytes(48))
    t = 1
    while True:
        b = t.to_bytes(48, "little") + bytes(48)
        if o.g2_deserialize(b, False) is not None and o.g2_deserialize(b, True) is None: break
        t += 1
    g2.append(b)
    return g1, g2


def popcount(bm, n): return sum(1 for i in range(n) if bm[i >> 3] >> (i & 7) & 1)


def generate():
    orc = Oracle()
    sks = [wl.sk_bytes(wl.seeded_sk(TAG, i)) for i in range(N_KEYS)]
    ski = [wl.seeded_sk(TAG, i) for i in range(N_KEYS)]
    pks = [orc.pk(k) for k in sks]
    msgs = [wl.seeded_bytes(TAG + "/msg", j, n) for j, n in enumerate(MSG_LENS)]
    hms = [orc.map(m) for m in msgs]
    assert all(hms)
    sigs = [orc.sign(sks[j], msgs[j]) for j in range(len(msgs))]
    t0 = bytes(32)
    assert orc.map(t0) is None
    # a hand-filled secret key >= Z^4 (plain ladder); its signature = (k mod r) * H(m)
    big = int.from_bytes(wl.seeded_bytes(TAG + "/big", 0, 32), "little") | (0xff << 248)
    assert big >= o.Z_ABS ** 4
    sig_big = orc.sign(wl.sk_bytes(big % wl.R_ORDER), msgs[3])
    g1r, g2r = reject_encodings()
    for b in g1r: assert not orc.pk_ok(b)
    for b in g2r: assert not orc.sig_ok(b)
    # field products on edge operands
    P = o.P
    ops = [0, 1, 2, P - 1, P - 2, (1 << 384) % P, 1 << 380, int.from_bytes(wl.seeded_bytes(TAG + "/fp", 0, 48), "little") % P]
    opb = [v.to_bytes(48, "little") for v in ops]
    prod = [orc.fp_mul(a, b) for a in opb for b in opb]
    # masks over the 16-key committee: empty, full, one key, and seeded ones
    bms = [bytes(2), b"\xff\xff", b"\x01\x00"] + [wl.bitmap_with_k(TAG + "/bm", j, N_KEYS, k) for j, k in enumerate([3, 8, 11, 12, 15])]
    bm_apk = [orc.mask_agg(pks, b) for b in bms]
    # committee rounds: 48-byte messages, signed with the summed key of the round's bitmap; then the reject classes
    rbm = [bytearray(wl.bitmap_with_k(TAG + "/round", j, N_KEYS, 9 + j % 8)) for j in range(N_ROUNDS)]
    rmsg = [bytearray(wl.seeded_bytes(TAG + "/round/m", j, 48)) for j in range(N_ROUNDS)]
    rsig = [bytearray(orc.sign(wl.sk_bytes(wl.round_signer_sum(ski, bytes(rbm[j]))), bytes(rmsg[j]))) for j in range(N_ROUNDS)]
    rsig[1], rsig[9] = rsig[9], rsig[1]           # swapped pair inside one group (group 1 of 4 and of 8)
    rmsg[2][17] ^= 0x20                           # wrong message
    rbm[5] = bytearray(2)                         # empty bitmap: identity key
    rsig[6] = bytearray(g2r[0])                   # x >= p
    rsig[10] = bytearray(g2r[2])                  # outside the subgroup
    rsig[13] = bytearray(g2r[1])                  # not on the curve
    rmsg[14] = bytearray(48)                      # t = 0: no H(m)
    rmsg[34][3] ^= 1                              # tail round, wrong message
    rok, rhdr = [], []
    for j in range(N_ROUNDS):
        ok = orc.agg_verify(pks, bytes(rbm[j]), bytes(rsig[j]), bytes(rmsg[j]))
        rok.append(1 if ok else 0)
        if not orc.sig_ok(bytes(rsig[j])): rhdr.append(3)
        elif popcount(rbm[j], N_KEYS) < QUORUM: rhdr.append(2)
        else: rhdr.append(1 if ok else 0)
    assert rok.count(0) == 9
    # votes of keys 0-5 on one 48-byte message (same-message batch, ballot box); vote 4 carries vote 5's signature
    vmsg = wl.seeded_bytes(TAG + "/vote", 0, 48)
    vsig = [orc.sign(sks[i], vmsg) for i in range(6)]
    vagg = orc.agg_sigs(vsig)
    vbm = [bytes([1 << i, 0]) for i in range(6)]
    vuse = list(vsig); vuse[4] = vsig[5]
    vok = [1 if orc.agg_verify(pks, vbm[i], vuse[i], vmsg) else 0 for i in range(6)]
    # independent triples (32-byte messages): six valid, then the reject classes
    tsk = [wl.sk_bytes(wl.seeded_sk(TAG + "/tri", i)) for i in range(12)]
    tpk = [orc.pk(k) for k in tsk]
    tmsg = [wl.seeded_bytes(TAG + "/tri/m", i, 32) for i in range(12)]
    tsig = [orc.sign(tsk[i], tmsg[i]) for i in range(12)]
    tpk[6] = g1r[0]                               # key x >= p
    tpk[7] = g1r[2]                               # key outside the subgroup
    tpk[8] = bytes(48); tsig[8] = bytes(96)       # identity key (and signature)
    tsig[9] = g2r[1]                              # signature not on the curve
    tsig[10] = tsig[11]                           # another key's signature
    tmsg[11] = t0                                 # t = 0
    tok, tst = [], []
    for i in range(12):
        ok = orc.verify(tsig[i], tpk[i], tmsg[i])
        tok.append(1 if ok else 0)
        tst.append(4 if not orc.pk_ok(tpk[i]) else 3 if not orc.sig_ok(tsig[i]) else (1 if ok else 0))
    # Part-1 VerifyHash turn: (signature, key, message) indices into sigs / pks / msgs, message 0 repeated
    p1 = [(0, 0, 0), (1, 1, 1), (0, 0, 0), (0, 1, 0), (2, 2, 0), (3, 3, 3), (5, 5, 5), (4, 4, 4), (0, 0, 3)]
    p1ok = [1 if orc.verify(sigs[s], pks[p], msgs[m]) else 0 for s, p, m in p1]
    return dict(sks=sks, pks=pks, msgs=msgs, hms=hms, sigs=sigs, big=big, sig_big=sig_big, g1r=g1r, g2r=g2r, opb=opb, prod=prod,
                pk_add=orc.pk_add(pks[0], pks[1], 0), pk_sub=orc.pk_add(pks[0], pks[1], 1), sig_add=orc.sig_add(sigs[0], sigs[1]),
                agg=orc.agg_sigs(sigs), bms=bms, bm_apk=bm_apk, rbm=rbm, rmsg=rmsg, rsig=rsig, rok=rok, rhdr=rhdr,
                tpk=tpk, tsig=tsig, tmsg=tmsg, tok=tok, tst=tst, p1=p1, p1ok=p1ok, vmsg=vmsg, vsig=vsig, vagg=vagg, vok=vok)


def c_bytes(b): return "{" + ",".join(f"0x{x:02x}" for x in b) + "}"
def c_arr(name, rows, width):
    lines = [f"static const uint8_t {name}[{len(rows)}][{width}] = {{"]
    for r in rows:
        assert len(r) == width, (name, len(r))
        lines.append("    " + c_bytes(r) + ",")
    return lines + ["};"]
def c_vec(name, b): return [f"static const uint8_t {name}[{len(b)}] = {c_bytes(b)};"]


def render(d):
    L = ["// GENERATED by oracle/gen_selftest.py -- do not edit.  Known answers of hbls_self_test (selftest.cuh).",
         f"// Inputs: harmony_b200/workload.py seeded_bytes / seeded_sk with tag \"{TAG}\" (\"{TAG}/msg\", \"{TAG}/round\", \"{TAG}/tri\", ...);",
         "// reject encodings: the first x = 1, 2, ... of each class (oracle/pyref.py).  Expected outputs: oracle/hbls_oracle.c.",
         "#pragma once", "#include <stdint.h>",
         f"#define ST_NKEYS {N_KEYS}", f"#define ST_NMSG {len(MSG_LENS)}", f"#define ST_NROUNDS {N_ROUNDS}", f"#define ST_QUORUM {QUORUM}",
         "#define ST_NTRI 12", f"#define ST_NP1 {len(d['p1'])}", f"#define ST_NBM {len(d['bms'])}"]
    L += c_arr("st_sk", d["sks"], 32) + c_arr("st_pk", d["pks"], 48)
    L += [f"static const uint32_t st_msg_len[{len(MSG_LENS)}] = {{{', '.join(map(str, MSG_LENS))}}};"]
    L += c_arr("st_msg", [m + bytes(64 - len(m)) for m in d["msgs"]], 64) + c_arr("st_hm", d["hms"], 96) + c_arr("st_sig", d["sigs"], 96)
    L += ["// secret-key struct >= Z^4 (plain ladder) and its signature of st_msg[3]"]
    L += c_vec("st_sk_big", d["big"].to_bytes(32, "little")) + c_vec("st_sig_big", d["sig_big"])
    L += ["// rejected encodings: [0] x >= p, [1] not on the curve, [2] outside the order-r subgroup"]
    L += c_arr("st_g1_rej", d["g1r"], 48) + c_arr("st_g2_rej", d["g2r"], 96)
    L += ["// field operands (canonical, little-endian) and their 64 products a[i] * b[j] at [8 i + j]"]
    L += c_arr("st_fp_op", d["opb"], 48) + c_arr("st_fp_prod", d["prod"], 48)
    L += ["// single-element ops: pk0 + pk1, pk0 - pk1, sig0 + sig1; sum of st_sig"]
    L += c_vec("st_pk_add", d["pk_add"]) + c_vec("st_pk_sub", d["pk_sub"]) + c_vec("st_sig_add", d["sig_add"]) + c_vec("st_sig_agg", d["agg"])
    L += ["// committee bitmaps (empty, full, one key, seeded) and their aggregate keys"]
    L += c_arr("st_bm", d["bms"], 2) + c_arr("st_bm_apk", d["bm_apk"], 48)
    L += ["// committee rounds: bitmap, signature, 48-byte message; verdict and header status (quorum ST_QUORUM)",
          "// rejects: 1/9 swapped signatures, 2 wrong message, 5 empty bitmap, 6 x >= p, 10 outside the subgroup, 13 off the curve,",
          "// 14 t = 0 message, 34 wrong message in the tail"]
    L += c_arr("st_rnd_bm", d["rbm"], 2) + c_arr("st_rnd_sig", d["rsig"], 96) + c_arr("st_rnd_msg", d["rmsg"], 48)
    L += c_vec("st_rnd_ok", bytes(d["rok"])) + c_vec("st_rnd_hdr", bytes(d["rhdr"]))
    L += ["// independent triples (32-byte messages): 0-5 valid, 6 key x >= p, 7 key outside the subgroup, 8 identity key,",
          "// 9 signature off the curve, 10 another key's signature, 11 t = 0 message; verdict and hbls_verify_batch_status code"]
    L += c_arr("st_tri_pk", d["tpk"], 48) + c_arr("st_tri_sig", d["tsig"], 96) + c_arr("st_tri_msg", d["tmsg"], 32)
    L += c_vec("st_tri_ok", bytes(d["tok"])) + c_vec("st_tri_status", bytes(d["tst"]))
    L += ["// Part-1 VerifyHash turn: {signature, key, message} indices into st_sig / st_pk / st_msg, and the verdicts"]
    L += [f"static const uint8_t st_p1[{len(d['p1'])}][3] = {{" + ", ".join("{%d,%d,%d}" % t for t in d["p1"]) + "};"]
    L += c_vec("st_p1_ok", bytes(d["p1ok"]))
    L += ["// votes of keys 0-5 on st_vote_msg, their sum, and the verdicts of the same-message batch in which vote 4 carries vote 5's",
          "// signature (bitmap of vote i: key i only)"]
    L += c_vec("st_vote_msg", d["vmsg"]) + c_arr("st_vote_sig", d["vsig"], 96) + c_vec("st_vote_agg", d["vagg"]) + c_vec("st_vote_ok", bytes(d["vok"]))
    return "\n".join(L) + "\n"


if __name__ == "__main__":
    text = render(generate())
    if "--check" in sys.argv:
        same = os.path.exists(OUT) and open(OUT).read() == text
        print("up to date" if same else "differs"); sys.exit(0 if same else 1)
    open(OUT, "w").write(text)
    print("wrote", OUT)
