"""Challenge and response files of a coordinated phase-1 ceremony on the host: their sizes and the power read back from
a size, and the pure-Python restatement (tests/challenge_oracle.py) against tests/phase1_oracle.py -- export, challenge
contribute and import give the same file as a direct contribution."""
import hashlib

import pytest

from distributed_groth16_b200 import formats
from distributed_groth16_b200.groth16 import phase2

SEED = [0xC3, 1, 2, 3, 4, 5, 6, 7]


@pytest.mark.parametrize("power", list(range(1, 28)))
def test_sizes_and_power_from_size(power):
    import challenge_oracle as co
    assert formats.ptau_challenge_bytes(power) == co.challenge_size(power) == 384 * (1 << power) + 128
    assert formats.ptau_response_bytes(power) == co.response_size(power) == 192 * (1 << power) + 864
    assert formats.ptau_challenge_power(formats.ptau_challenge_bytes(power)) == power
    assert formats.ptau_response_power(formats.ptau_response_bytes(power)) == power
    for d in (-1, 1):
        with pytest.raises(formats.FormatError):
            formats.ptau_challenge_power(formats.ptau_challenge_bytes(power) + d)
        with pytest.raises(formats.FormatError):
            formats.ptau_response_power(formats.ptau_response_bytes(power) + d)


def test_sizes_outside_the_powers():
    for size in (0, 64, formats.ptau_challenge_bytes(0), formats.ptau_challenge_bytes(28)):
        with pytest.raises(formats.FormatError):
            formats.ptau_challenge_power(size)
    for size in (0, 864, formats.ptau_response_bytes(0), formats.ptau_response_bytes(28)):
        with pytest.raises(formats.FormatError):
            formats.ptau_response_power(size)


@pytest.mark.parametrize("power", [1, 2])
def test_challenge_round_equals_a_contribution(power):
    """export -> challenge contribute (rng A) -> import (name N) == phase1_oracle.contribute(P, rng A, N), twice in a row;
    Blake2b of the challenge is the file's current challenge and Blake2b of the response is the responseHash."""
    import challenge_oracle as co
    import phase1_oracle as po
    p0 = po.new(power)
    ch0 = co.export_challenge(p0)
    assert len(ch0) == formats.ptau_challenge_bytes(power)
    assert ch0[:64] == hashlib.blake2b(b"", digest_size=64).digest()
    assert hashlib.blake2b(ch0, digest_size=64).digest() == po.first_challenge_hash(power)
    resp, ch_hash, rh = co.challenge_contribute(ch0, phase2.ChaCha(SEED))
    assert ch_hash == po.first_challenge_hash(power)
    assert len(resp) == formats.ptau_response_bytes(power)
    assert resp[:64] == ch_hash and hashlib.blake2b(resp, digest_size=64).digest() == rh
    p1, irh, inc = co.import_response(p0, resp, name="remote")
    want, wrh, wnc = po.contribute(p0, phase2.ChaCha(SEED), name="remote")
    assert (irh, inc) == (wrh, wnc) == (rh, wnc)
    assert p1 == want
    # a second round from the imported file: the challenge now starts with the first responseHash
    ch1 = co.export_challenge(p1)
    assert ch1[:64] == wrh
    assert hashlib.blake2b(ch1, digest_size=64).digest() == wnc
    seed2 = [0xD4] + SEED[1:]
    resp2, _, rh2 = co.challenge_contribute(ch1, phase2.ChaCha(seed2))
    p2, irh2, _ = co.import_response(p1, resp2)
    want2, wrh2, _ = po.contribute(p1, phase2.ChaCha(seed2))
    assert irh2 == wrh2 == rh2
    assert p2 == want2
