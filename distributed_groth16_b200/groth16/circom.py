"""Circom / snarkjs artefacts -> device-resident prover inputs, and the one-call prover on top of them
(the flow of /root/reference/groth16/examples/sha256.rs:127-169 and mpc-api/src/main.rs:282-421 minus the
WASM witness calculator: the witness comes from a .wtns file or from the caller)."""
from __future__ import annotations

import numpy as np

from .. import formats
from ..context import Net
from . import prove
from .proving_key import ProvingKey
from .qap import ConstraintMatrices, qap


def load_zkey(net: Net, zkey_bytes: bytes):
    """-> (ProvingKey resident in HBM, ConstraintMatrices, formats.ZKey)   (ark-circom/src/zkey.rs:53-60)."""
    zk = formats.read_zkey(zkey_bytes)
    pk = ProvingKey(net, zk.a_query, zk.b_g1_query, zk.b_g2_query, zk.l_query, zk.h_query, zk.n_inputs, zk.alpha_g1,
                    zk.beta_g1, zk.delta_g1, zk.beta_g2, zk.delta_g2)
    coo = []
    for mi in (0, 1):
        sel = zk.coef_matrix == mi
        coo.append((zk.coef_row[sel], zk.coef_col[sel], zk.coef_val_r2[sel]))
    mats = ConstraintMatrices(net, zk.n_inputs, zk.num_constraints, coo[0], coo[1], values_montgomery_depth=1)
    return pk, mats, zk


def ptau_prepare_phase2(net: Net, src_path: str, dst_path: str) -> None:
    """snarkjs `powersoftau prepare phase2 <src> <dst>` on the GPU: the Lagrange sections 12-15 that zkey_new reads, computed
    from the tau-power sections of a phase-1 ceremony file and streamed to dst_path (ptau.prepare_phase2)."""
    from . import ptau
    ptau.prepare_phase2(net, src_path, dst_path)


def ptau_new(path: str, power: int) -> None:
    """snarkjs `powersoftau new bn128 <power>` (power 1..27): a phase-1 ceremony file with the generators in every slot
    and no contributions (phase1.new; file writing only)."""
    from . import phase1
    phase1.new(path, power)


def ptau_contribute(net: Net, src_path: str, dst_path: str, name: str | None = None, entropy: str = ""):
    """snarkjs `powersoftau contribute <src> <dst>` on the GPU: the key is drawn, as snarkjs getRandomRng does, from a
    ChaCha seeded with Blake2b-512(os.urandom(64) || UTF-8 entropy); the secrets are dropped on return.  Returns
    (responseHash, nextChallenge)."""
    import hashlib
    import os
    from . import phase1, phase2
    rng = phase2.ChaCha.from_hash(hashlib.blake2b(os.urandom(64) + str(entropy).encode("utf-8"), digest_size=64).digest())
    return phase1.contribute(net, src_path, dst_path, rng, name=name)


def ptau_beacon(net: Net, src_path: str, dst_path: str, beacon_hash: bytes, num_iterations_exp: int,
                name: str | None = None):
    """snarkjs `powersoftau beacon <src> <dst> <hash> <e>`: the final, publicly reproducible contribution (2^e SHA-256
    rounds on the host).  Returns (responseHash, nextChallenge)."""
    from . import phase1
    if not 10 <= int(num_iterations_exp) <= 63:
        raise ValueError("num_iterations_exp must be in 10..63, got %d" % num_iterations_exp)
    if len(beacon_hash) > 255:
        raise ValueError("beacon hash longer than 255 bytes")
    return phase1.beacon(net, src_path, dst_path, bytes(beacon_hash), int(num_iterations_exp), name=name)


def ptau_export_challenge(net: Net, ptau_path: str, challenge_path: str) -> bytes:
    """snarkjs `powersoftau export challenge <ptau> <challenge>`: the bare challenge a contributor works on, without the
    .ptau (phase1.export_challenge).  Returns the challenge hash."""
    from . import phase1
    return phase1.export_challenge(net, ptau_path, challenge_path)


def ptau_challenge_contribute(net: Net, challenge_path: str, response_path: str, entropy: str = ""):
    """snarkjs `powersoftau challenge contribute bn128 <challenge> <response>` on the GPU, the key drawn as in
    ptau_contribute; the secrets are dropped on return.  Returns (challengeHash, responseHash)."""
    import hashlib
    import os
    from . import phase1, phase2
    rng = phase2.ChaCha.from_hash(hashlib.blake2b(os.urandom(64) + str(entropy).encode("utf-8"), digest_size=64).digest())
    return phase1.challenge_contribute(net, challenge_path, response_path, rng)


def ptau_import_response(net: Net, ptau_path: str, response_path: str, dst_path: str, name: str | None = None):
    """snarkjs `powersoftau import response <ptau> <response> <dst>`: the contributor's response appended to the ceremony
    as a new record (phase1.import_response; it does not verify, ptau_verify does).  Returns (responseHash,
    nextChallenge)."""
    from . import phase1
    return phase1.import_response(net, ptau_path, response_path, dst_path, name=name)


def ptau_verify(net: Net, ptau_path: str):
    """snarkjs `powersoftau verify <ptau>` on the GPU: -> phase1.Phase1Report (ok, one failure line per check that does
    not hold, naming the contribution or section; per record its name, type and nextChallenge)."""
    from . import phase1
    return phase1.verify(net, ptau_path)


def ptau_check_lagrange(net: Net, ptau_path: str):
    """The Lagrange part of snarkjs `powersoftau verify` on a prepared file: -> ptau.LagrangeReport (ok, one failure line
    per section and level that does not check).  Needs no toxic waste."""
    from . import ptau
    return ptau.check_lagrange(net, ptau_path)


def zkey_new(net: Net, r1cs_bytes: bytes, ptau_path: str, cs_hash: bool = False) -> bytes:
    """snarkjs `zkey new <r1cs> <ptau>` on the GPU (scripts/phase2_proving_key.sh, ark-circom/test-vectors/complex-circuit/
    build.sh:11): the .zkey bytes of the circuit's proving key from a prepared Powers-of-Tau file.  The key has delta = 1:
    it needs a phase-2 contribution before production use.  Section 10 starts with a zero csHash (formats.write_zkey)
    unless cs_hash is True; then it holds the circuit hash snarkjs writes (cshash.cs_hash), and every other byte is the
    same."""
    with formats.read_ptau(ptau_path) as pt:
        return zkey_from_r1cs(net, formats.read_r1cs(r1cs_bytes), pt, cs_hash=cs_hash)


def zkey_cs_hash(net: Net, r1cs_bytes: bytes, ptau_path: str) -> bytes:
    """The circuit hash (csHash) of the circuit's `zkey new` key from a prepared Powers-of-Tau file: the 64 bytes snarkjs
    prints as "Circuit hash" and stores at the start of zkey section 10 (cshash.cs_hash)."""
    from .cshash import cs_hash
    from .setup import ptau_key_points
    with formats.read_ptau(ptau_path) as pt:
        return cs_hash(net, ptau_key_points(net, formats.read_r1cs(r1cs_bytes), pt), pt)


def _random_scalar(entropy: bytes) -> int:
    """A non-zero scalar mod r from os.urandom mixed with the caller's entropy through Blake2b-512."""
    import hashlib
    import os
    while True:
        v = int.from_bytes(hashlib.blake2b(os.urandom(64) + bytes(entropy), digest_size=64).digest(), "little") % formats.FR_MODULUS
        if v:
            return v


def zkey_contribute(net: Net, zkey_bytes: bytes, name: str | None = None, entropy: bytes = b""):
    """snarkjs `zkey contribute` on the GPU (scripts/phase2_proving_key.sh): a phase-2 contribution with a fresh secret x
    (os.urandom mixed with `entropy` through Blake2b) and proof-of-knowledge base g1_s = s G for a fresh s.  L and H are
    multiplied by x^-1 on the device.  The secrets are dropped on return.  Returns (zkey bytes, contribution hash)."""
    from . import phase2
    x, s = _random_scalar(entropy), _random_scalar(entropy)
    g1_s = phase2._scale_one(net, np.concatenate([_fq_mont_limbs(1), _fq_mont_limbs(2)]), s)
    return phase2.contribute(net, zkey_bytes, x, g1_s, name=name)


def _fq_mont_limbs(v: int) -> np.ndarray:
    x = v * (1 << 256) % formats.FQ_MODULUS
    return np.array([(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def zkey_beacon(net: Net, zkey_bytes: bytes, beacon_hash: bytes, num_iterations_exp: int, name: str | None = None):
    """snarkjs `zkey beacon`: the final, publicly reproducible contribution from a beacon value (2^num_iterations_exp
    SHA-256 rounds on the host, so large exponents take long).  Returns (zkey bytes, contribution hash)."""
    from . import phase2
    if not 10 <= int(num_iterations_exp) <= 63:
        raise ValueError("num_iterations_exp must be in 10..63, got %d" % num_iterations_exp)
    if len(beacon_hash) > 255:
        raise ValueError("beacon hash longer than 255 bytes")
    return phase2.beacon(net, zkey_bytes, bytes(beacon_hash), int(num_iterations_exp), name=name)


def zkey_verify(net: Net, r1cs_bytes: bytes, ptau_path: str, zkey_bytes: bytes, check_cs_hash: bool = False):
    """snarkjs `zkey verify <r1cs> <ptau> <zkey>`: -> phase2.Phase2Report (ok, failure reasons, per contribution its name,
    type and hash, and the csHash found in the file).  check_cs_hash also recomputes the circuit hash from the circuit and
    the ceremony and fails when the file's differs, as snarkjs does; without it the csHash is carried, not checked."""
    from . import phase2
    return phase2.verify(net, r1cs_bytes, ptau_path, zkey_bytes, check_cs_hash=check_cs_hash)


def zkey_export_bellman(net: Net, zkey_bytes: bytes) -> bytes:
    """snarkjs `zkey export bellman <zkey> <params>`: the bellman MPC-params bytes a coordinated phase-2 ceremony sends to
    its contributors, with the H query moved to the tau basis on the device (bellman.export).  Domains up to 2^27."""
    from . import bellman
    return bellman.export(net, zkey_bytes)


def zkey_bellman_contribute(net: Net, challenge_bytes: bytes, entropy: bytes = b""):
    """snarkjs `zkey bellman contribute bn128 <challenge> <response>` on the GPU, with a fresh secret x and base g1_s as in
    zkey_contribute; the secrets are dropped on return.  Returns (response bytes, contribution hash)."""
    from . import bellman, phase2
    x, s = _random_scalar(entropy), _random_scalar(entropy)
    g1_s = phase2._scale_one(net, np.concatenate([_fq_mont_limbs(1), _fq_mont_limbs(2)]), s)
    return bellman.contribute(net, challenge_bytes, x, g1_s)


def zkey_import_bellman(net: Net, zkey_bytes: bytes, response_bytes: bytes, name: str | None = None) -> bytes:
    """snarkjs `zkey import bellman <zkey> <response> <dst>`: the key with the response's contributions applied, the new
    records named `name` (bellman.import_response).  It checks that the response answers this key but runs no pairing
    check: run zkey_verify on the result."""
    from . import bellman
    return bellman.import_response(net, zkey_bytes, response_bytes, name=name)


def zkey_from_r1cs(net: Net, r1: formats.R1CS, pt: formats.PTau, cs_hash: bool = False) -> bytes:
    """zkey_new on a parsed r1cs and an open ceremony file."""
    import struct
    from .setup import ptau_key_points
    q = ptau_key_points(net, r1, pt)
    sec10 = None
    if cs_hash:
        from .cshash import cs_hash as circuit_hash
        sec10 = circuit_hash(net, q, pt) + struct.pack("<I", 0)
    r2 = lambda i: net.fr_convert(net.to_device(np.ascontiguousarray(r1.vals[i], dtype=np.uint64).reshape(-1, 4)),
                                  to_mont=True, times=2).cpu().numpy().view(np.uint64)     # value * R^2, on the device
    mi, ci, si, vi = formats.zkey_coefficients(q["n_public"], r1.n_constraints, (r1.rows[0], r1.cols[0], r2(0)),
                                               (r1.rows[1], r1.cols[1], r2(1)))
    host = lambda t: t.cpu().numpy().view(np.uint64)
    zk = formats.ZKey(n_vars=q["n_vars"], n_public=q["n_public"], domain_size=q["domain_size"], alpha_g1=q["alpha_g1"],
                      beta_g1=q["beta_g1"], beta_g2=q["beta_g2"], gamma_g2=q["gamma_g2"], delta_g1=q["delta_g1"],
                      delta_g2=q["delta_g2"], ic=host(q["ic"]), a_query=host(q["a_query"]), b_g1_query=host(q["b_g1_query"]),
                      b_g2_query=host(q["b_g2_query"]), l_query=host(q["l_query"]), h_query=host(q["h_query"]),
                      coef_matrix=mi, coef_row=ci, coef_col=si, coef_val_r2=vi)
    return formats.write_zkey(zk, section10=sec10)


def load_witness(net: Net, wtns_bytes: bytes):
    """.wtns -> full assignment z on the device in Montgomery form (wire index == witness index: the reference
    disables the wire mapping, ark-circom/src/circom/builder.rs:63-64)."""
    w = formats.read_wtns(wtns_bytes)
    return net.fr_convert(net.to_device(w), to_mont=True)


def witness_from_ints(net: Net, values):
    """canonical Python ints -> Montgomery device tensor (conversion on the GPU)."""
    arr = np.array([[(int(v) >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)] for v in values], dtype=np.uint64)
    return net.fr_convert(net.to_device(arr), to_mont=True)


def prove_from_matrices(pk: ProvingKey, matrices: ConstraintMatrices, z, r=None, s=None, mirror_reference_bg1=False) -> bytes:
    """qap() -> h -> MSMs -> 128 proof bytes, everything resident on the GPU
    (== Groth16::create_proof_with_reduction_and_matrices + serialize, sha256.rs:159-168)."""
    q = qap(matrices, z, pk.net)
    return prove.create_proof_dev(pk, z, q.a, q.b, q.c, r, s, mirror_reference_bg1)


def prove_zkey_wtns(net: Net, zkey_bytes: bytes, wtns_bytes: bytes, r=None, s=None):
    """-> (proof bytes, public inputs as canonical limbs (n_public, 4))."""
    pk, mats, zk = load_zkey(net, zkey_bytes)
    w = formats.read_wtns(wtns_bytes)
    if w.shape[0] != zk.n_vars:
        raise formats.FormatError("witness has %d entries, the key expects %d" % (w.shape[0], zk.n_vars))
    z = net.fr_convert(net.to_device(w), to_mont=True)
    proof = prove_from_matrices(pk, mats, z, r, s)
    pk.free()
    return proof, w[1:1 + zk.n_public].copy()


def wtns_check(net: Net, r1cs_bytes: bytes, wtns_bytes: bytes):
    """snarkjs `wtns check <r1cs> <wtns>`: does the witness satisfy the circuit?  -> snarkjs.WtnsCheckReport (ok, n_failed,
    first_failed, one line per failure).  A witness whose length is not the circuit's wire count, whose w[0] is not 1 or
    with an entry >= r fails with one line naming the index; otherwise every constraint <A_i,w> <B_i,w> = <C_i,w> is
    evaluated on the device, and the line for the first failing one gives its three products."""
    from . import snarkjs
    return snarkjs.check_witness(net, formats.read_r1cs(r1cs_bytes), formats.read_wtns(wtns_bytes))


def zkey_export_verificationkey(net: Net, zkey_bytes: bytes) -> str:
    """snarkjs `zkey export verificationkey <zkey> <json>`: the text of verification_key.json, vk_alphabeta_12 computed on
    the device."""
    from . import snarkjs
    return formats.write_vk_json(snarkjs.vk_from_zkey(net, formats.read_zkey(zkey_bytes)))


def groth16_prove(net: Net, zkey_bytes: bytes, wtns_bytes: bytes, r=None, s=None):
    """snarkjs `groth16 prove <zkey> <wtns> <proof.json> <public.json>`: prove_zkey_wtns (r, s as it takes them: 4 Montgomery
    limbs each, None = 0), written as snarkjs writes it.  -> (text of proof.json, text of public.json)."""
    from . import snarkjs
    proof, public = prove_zkey_wtns(net, zkey_bytes, wtns_bytes, r, s)
    return snarkjs.proof_to_json(net, proof), snarkjs.public_to_json(public)


def groth16_verify(net: Net, vk_json, public_json, proof_json) -> bool:
    """snarkjs `groth16 verify <verification_key.json> <public.json> <proof.json>` on the texts of the three files.
    Raises formats.FormatError for a malformed file (not JSON, a missing key, protocol other than groth16 or curve other than
    bn128, a non-numeric string, a coordinate >= q, a verification-key point that does not decode, len(IC) != nPublic + 1).
    Returns False where snarkjs does: a public count other than nPublic, a signal >= r, a proof point off the curve or
    outside the G2 subgroup, or a failing pairing check."""
    from . import snarkjs
    return snarkjs.verify_json(net, vk_json, public_json, proof_json)
