"""Pure-Python restatement of snarkjs `zkey new` for tiny circuits (TEST INFRASTRUCTURE ONLY): r1cs bytes + prepared ptau
bytes -> zkey bytes, with the oracle's group law and its own reading of both files.  It is the yardstick of
distributed_groth16_b200.groth16.circom.zkey_new.  With L, L2, alpha L, beta L the Lagrange bases of the circuit's domain
2^k and H those of 2^(k+1) (the ptau layout of tests/ptau_writer.py):

  A[s] = sum_c A[c,s] L_c + [s <= n_public] L_{nc+s}        B1[s] / B2[s] = sum_c B[c,s] L_c / L2_c
  K[s] = sum_c (A[c,s] beta L_c + B[c,s] alpha L_c + C[c,s] L_c) + [s <= n_public] beta L_{nc+s}
  IC = K[:n_public + 1], C section = K[n_public + 1:], H[i] = H_{2i+1}
  header: alpha_1, beta_1, beta_2 from the ptau, gamma_2 = delta_2 = the G2 generator, delta_1 = the G1 generator."""
import struct

from artefact_writer import Q, R, container
from oracle import bn254 as o, layout


def zkey_new(r1cs_bytes: bytes, ptau: bytes) -> bytes:
    r1 = o.read_r1cs(r1cs_bytes)
    secs = o._sections(ptau, b"ptau")
    nc, n_vars = r1["n_constraints"], r1["n_wires"]
    n_public = r1["n_pub_out"] + r1["n_pub_in"]
    k = 0
    while (1 << k) < nc + n_public + 1:
        k += 1
    m = 1 << k

    def level(sid, lv, g2=False):
        w = 128 if g2 else 64
        off = secs[sid][0][0] + ((1 << lv) - 1) * w
        rd = o._rd_g2 if g2 else o._rd_g1
        return [rd(ptau, off + i * w) for i in range(1 << lv)]

    L, L2, aL, bL = level(12, k), level(13, k, True), level(14, k), level(15, k)
    H = level(12, k + 1)[1::2]
    first = lambda sid, g2=False: (o._rd_g2 if g2 else o._rd_g1)(ptau, secs[sid][0][0])
    A, B1, K = [None] * n_vars, [None] * n_vars, [None] * n_vars
    B2 = [None] * n_vars
    acc = lambda pts, s, base, v, G=o.G1: pts.__setitem__(s, G.add(pts[s], G.mul(base, v)))
    coefs = []
    for c, (la, lb, lc) in enumerate(r1["constraints"]):
        for v, s in la:
            acc(A, s, L[c], v)
            acc(K, s, bL[c], v)
            coefs.append((0, c, s, v))
        for v, s in lb:
            acc(B1, s, L[c], v)
            acc(B2, s, L2[c], v, o.G2)
            acc(K, s, aL[c], v)
            coefs.append((1, c, s, v))
        for v, s in lc:
            acc(K, s, L[c], v)
    for j in range(n_public + 1):
        acc(A, j, L[nc + j], 1)
        acc(K, j, bL[nc + j], 1)
        coefs.append((0, nc + j, j, 1))
    g1 = lambda pts: layout.g1_to_arr(pts).tobytes()
    g2 = lambda pts: layout.g2_to_arr(pts).tobytes()
    hdr = struct.pack("<I", 32) + Q.to_bytes(32, "little") + struct.pack("<I", 32) + R.to_bytes(32, "little")
    hdr += struct.pack("<III", n_vars, n_public, m)
    hdr += g1([first(4), first(5)]) + g2([first(6, True), o.G2_GEN]) + g1([o.G1_GEN]) + g2([o.G2_GEN])
    r2 = o.MONT_R * o.MONT_R % R
    sec4 = struct.pack("<I", len(coefs)) + b"".join(struct.pack("<III", mi, c, s) + (v * r2 % R).to_bytes(32, "little")
                                                    for mi, c, s, v in coefs)
    body = {1: struct.pack("<I", 1), 2: hdr, 3: g1(K[:n_public + 1]), 4: sec4, 5: g1(A), 6: g1(B1), 7: g2(B2),
            8: g1(K[n_public + 1:]), 9: g1(H), 10: bytes(64) + struct.pack("<I", 0)}
    return container(b"zkey", [(sid, body[sid]) for sid in (1, 2, 4, 3, 9, 8, 5, 6, 7, 10)])
