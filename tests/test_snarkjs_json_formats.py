"""snarkjs's Groth16 JSON files as text (distributed_groth16_b200/formats.py): proof.json, public.json and
verification_key.json, pinned against the files snarkjs wrote for the reference's million-constraint circuit.
tests/golden/snarkjs_million/ holds the reference's fixtures/million/{proof,public,verification_key}.json copied byte for
byte (data only; the same triple that tests/golden/reference_goldens.json carries as parsed JSON).  CPU only."""
import json
import os

import pytest

from distributed_groth16_b200 import formats

M = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "snarkjs_million")
FILES = {"proof.json": (formats.read_proof_json, formats.write_proof_json),
         "public.json": (formats.read_public_json, formats.write_public_json),
         "verification_key.json": (formats.read_vk_json, formats.write_vk_json)}


def _text(name):
    return open(os.path.join(M, name)).read()


@pytest.mark.parametrize("name", sorted(FILES))
def test_reading_and_writing_each_million_file_reproduces_it_byte_for_byte(name):
    rd, wr = FILES[name]
    raw = open(os.path.join(M, name), "rb").read()
    assert wr(rd(raw.decode())).encode() == raw
    assert not raw.endswith(b"\n")


def test_the_million_files_read_as_expected():
    vk = formats.read_vk_json(_text("verification_key.json"))
    assert vk.n_public == 1 and len(vk.ic) == 2 and vk.gamma_2 == vk.delta_2
    assert vk.alpha_1[0] == 20491192805390485299153009773594534940189261866228447918068658471970481763042
    assert vk.beta_2[0] == (6375614351688725206403948262868962793625744043794305715222011528459656738731,
                            4252822878758300859123897981450591353533073413197771768651442665752259397132)
    assert vk.alphabeta_12[1][2][1] == 8037395052364110730298837004334506829870972346962140206007064471173334027475
    assert formats.read_public_json(_text("public.json")) == [999992]
    pr = formats.read_proof_json(_text("proof.json"))
    assert pr.pi_a[1] == 4467227993235159900656781320247733325074718480281314529638990710876350942641


def test_hex_strings_are_accepted():
    obj = json.loads(_text("proof.json"))
    obj["pi_a"] = [hex(int(v)) for v in obj["pi_a"]]
    obj["pi_b"][0] = ["0x" + format(int(v), "X") for v in obj["pi_b"][0]]
    hexed = formats.read_proof_json(json.dumps(obj))
    assert hexed == formats.read_proof_json(_text("proof.json"))
    assert formats.write_proof_json(hexed) == _text("proof.json")
    assert formats.read_public_json('["0xf4238"]') == [999992]


def test_infinity_forms():
    p = formats.SnarkjsProof(None, None, None)
    obj = json.loads(formats.write_proof_json(p))
    assert obj["pi_a"] == ["0", "1", "0"] and obj["pi_b"] == [["0", "0"], ["1", "0"], ["0", "0"]]
    assert formats.read_proof_json(formats.write_proof_json(p)) == p
    assert formats.write_public_json([]) == "[]" and formats.read_public_json("[]") == []


def _mutated(name, fn):
    obj = json.loads(_text(name))
    fn(obj)
    return json.dumps(obj, indent=1)


def _set(path, value):
    def f(obj):
        o = obj
        for k in path[:-1]:
            o = o[k]
        o[path[-1]] = value
    return f


def _del(key):
    return lambda obj: obj.pop(key)


Q = formats.FQ_MODULUS
MALFORMED = [
    ("proof.json", lambda o: None, "{not json", "not JSON"),
    ("verification_key.json", lambda o: None, "[1, 2", "not JSON"),
    ("public.json", lambda o: None, "{]", "not JSON"),
    ("proof.json", _del("pi_c"), None, "pi_c"),
    ("proof.json", _del("protocol"), None, "protocol"),
    ("verification_key.json", _del("IC"), None, "IC"),
    ("verification_key.json", _del("vk_alphabeta_12"), None, "vk_alphabeta_12"),
    ("proof.json", _set(["protocol"], "plonk"), None, "protocol"),
    ("proof.json", _set(["curve"], "bls12381"), None, "curve"),
    ("verification_key.json", _set(["protocol"], "fflonk"), None, "protocol"),
    ("verification_key.json", _set(["curve"], "bls12381"), None, "curve"),
    ("proof.json", _set(["pi_a", 0], "12ab"), None, "pi_a[0]"),
    ("proof.json", _set(["pi_b", 1, 0], "-5"), None, "pi_b[1][0]"),
    ("proof.json", _set(["pi_c", 1], 7), None, "pi_c[1]"),
    ("public.json", _set([0], "99 99"), None, "public[0]"),
    ("proof.json", _set(["pi_a", 0], str(Q)), None, "pi_a[0]"),
    ("proof.json", _set(["pi_b", 0, 1], hex(Q + 5)), None, "pi_b[0][1]"),
    ("verification_key.json", _set(["vk_alpha_1", 1], str(Q)), None, "vk_alpha_1[1]"),
    ("verification_key.json", _set(["vk_alphabeta_12", 1, 2, 0], str(Q)), None, "vk_alphabeta_12[1][2][0]"),
    ("verification_key.json", _set(["IC", 1, 0], str(Q + 1)), None, "IC[1][0]"),
    ("proof.json", _set(["pi_a", 2], "2"), None, "pi_a"),
    ("proof.json", _set(["pi_b", 2], ["1", "1"]), None, "pi_b"),
    ("verification_key.json", _set(["vk_delta_2", 2], ["0", "1"]), None, "vk_delta_2"),
    ("verification_key.json", _set(["IC", 0, 2], "5"), None, "IC[0]"),
    ("verification_key.json", _set(["nPublic"], 2), None, "IC"),
    ("verification_key.json", lambda o: o["IC"].append(o["IC"][0]), None, "IC"),
    ("verification_key.json", _set(["nPublic"], "1"), None, "nPublic"),
]


@pytest.mark.parametrize("case", range(len(MALFORMED)))
def test_each_malformed_kind_raises_format_error_naming_the_field(case):
    name, fn, raw, field = MALFORMED[case]
    text = raw if raw is not None else _mutated(name, fn)
    with pytest.raises(formats.FormatError) as e:
        FILES[name][0](text)
    assert field in str(e.value)


def _writes_like_snarkjs(text_of, name):
    return text_of(FILES[name][0](_text(name))) == _text(name)


def test_mutant_writers_fail_the_round_trip():
    """The byte-for-byte test must catch each way a writer could plausibly go wrong."""
    assert _writes_like_snarkjs(formats.write_vk_json, "verification_key.json")
    swap = lambda p: None if p is None else ((p[0][1], p[0][0]), (p[1][1], p[1][0]))
    c1_first = lambda pr: formats.write_proof_json(formats.SnarkjsProof(pr.pi_a, swap(pr.pi_b), pr.pi_c))
    assert not _writes_like_snarkjs(c1_first, "proof.json")
    assert not _writes_like_snarkjs(lambda v: formats.write_public_json(v) + "\n", "public.json")
    assert not _writes_like_snarkjs(lambda v: json.dumps(json.loads(formats.write_vk_json(v)), indent=2),
                                    "verification_key.json")
