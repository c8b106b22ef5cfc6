"""Host mirror of InnerProductArgPC::open's halving loop (ipa_pc/mod.rs:612-722) over the device-resident
round kernels.  Names follow the reference (`compute_random_oracle_challenge`, `round_challenge`, `l_vec`,
`r_vec`, `final_comm_key`, `c`).

Transcript: exactly the reference's.  Every round hashes  round_challenge.serialize_uncompressed() ||
l.serialize_uncompressed() || r.serialize_uncompressed()  (:681-688) -- 32 little-endian canonical bytes for the scalar,
the curve's uncompressed point encoding (csrc/wire.cuh, produced on the device by pcgpu_g1_serialize) for l and r -- with
Blake2s-256 (the digest the reference's tests instantiate) and maps the digest to a scalar with Field::from_random_bytes
(ark-ff: keep MODULUS_BIT_SIZE bits of the little-endian digest, reject values >= r), retrying with an incremented
little-endian u64 counter appended (:74-87).  ark-serialize / ark-ff are un-vendored: restated from their published
behaviour (DESIGN.md section 2 lists what pins them).
"""
import hashlib

import numpy as np

from .binding import fq_limbs

_MODULI = {
    0: 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001,
    1: 21888242871839275222246405745257275088548364400416034343698204186575808495617,
    2: 0x40000000000000000000000000000000224698fc0994a8dd8c46eb2100000001,
}


def _fr_mont(curve, v):
    r = _MODULI[curve]
    m = v * (1 << 256) % r
    return np.array([(m >> (64 * j)) & (2**64 - 1) for j in range(4)], dtype=np.uint64)


def from_random_bytes(curve, digest):
    """Field::from_random_bytes for Fr (ark-ff Fp::from_random_bytes_with_flags::<EmptyFlags>): the 32 digest bytes as a
    little-endian integer with the bits above MODULUS_BIT_SIZE cleared; None unless the result is a reduced element"""
    r = _MODULI[curve]
    v = int.from_bytes(digest[:32], "little") & ((1 << r.bit_length()) - 1)
    return v if v < r else None


def compute_random_oracle_challenge(curve, data):
    """ipa_pc/mod.rs:74-87 with Blake2s-256 (the digest the reference's tests instantiate, ipa_pc/mod.rs:1051+)."""
    i = 0
    while True:
        v = from_random_bytes(curve, hashlib.blake2s(data + i.to_bytes(8, "little")).digest())
        if v is not None:
            return v
        i += 1


def round_transcript(eng, curve, round_challenge, l, l_inf, r, r_inf):
    """the bytes hashed for the next round challenge (:681-687)"""
    pts = np.stack([np.asarray(l, dtype=np.uint64).reshape(-1), np.asarray(r, dtype=np.uint64).reshape(-1)])
    enc = eng.g1_serialize(curve, pts, np.array([l_inf, r_inf], dtype=np.uint8), compressed=False)
    return int(round_challenge).to_bytes(32, "little") + enc.tobytes()


def open_rounds(eng, curve, comm_key_xy, coeffs, point, h_prime_xy, round_challenge, n=None, flags=0, n_coeffs=None,
                on_round=None):
    """The `while n > 1` loop (:665-711).  comm_key_xy: n affine points; coeffs: <= n Montgomery Fr; point: Montgomery
    Fr; h_prime_xy: affine h' = h * round_challenge (:631); round_challenge: the initial challenge as an int.  n, flags,
    n_coeffs: as Engine.ipa_begin (device-resident key and coefficients with DEVICE_PTRS).  on_round(t): called after
    round t's l and r are computed, before its fold.  Returns dict(l_vec, r_vec, final_comm_key, c, challenges)."""
    r = _MODULI[curve]
    st = eng.ipa_begin(curve, comm_key_xy, coeffs, point, n=n, flags=flags, n_coeffs=n_coeffs)
    l_vec, r_vec, chals = [], [], []
    while eng.ipa_len(st) > 1:
        l, l_inf, rr, r_inf = eng.ipa_round_lr(curve, st, h_prime_xy, with_inf=True)
        if on_round:
            on_round(len(l_vec))
        l_vec.append(l)
        r_vec.append(rr)
        data = round_transcript(eng, curve, round_challenge, l, l_inf, rr, r_inf)          # :681-687
        round_challenge = compute_random_oracle_challenge(curve, data)
        chals.append(round_challenge)
        inv = pow(round_challenge, -1, r)                                                    # :689
        eng.ipa_round_fold(st, _fr_mont(curve, round_challenge), _fr_mont(curve, inv))      # :691-708
    final_key, c = eng.ipa_finish(curve, st)
    return dict(l_vec=l_vec, r_vec=r_vec, final_comm_key=final_key, c=c, challenges=chals)


def check_final_key(eng, curve, comm_key_xy, challenges):
    """InnerProductArgPC::check's linear-time step (ipa_pc/mod.rs:760-766): the key the verifier recomputes from the round
    challenges, cm_commit(vk.comm_key, check_poly.compute_coeffs()) -- must equal proof.final_comm_key."""
    srs = eng.srs_register(curve, comm_key_xy)
    ch = np.stack([_fr_mont(curve, int(c)) for c in challenges])
    out = eng.ipa_check_final_key(srs, ch)
    srs.release()
    return out
