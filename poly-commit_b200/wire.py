"""Host mirror of the kzg10 containers' CanonicalSerialize / CanonicalDeserialize (SURVEY.md section 8f rank 1).

  Powers          kzg10/data_structures.rs:142-177   powers_of_g: Vec<G1Affine>, powers_of_gamma_g: Vec<G1Affine>
  Commitment      kzg10/data_structures.rs:315-328   one G1Affine (derived impl)
  Proof           kzg10/data_structures.rs:479-495   w: G1Affine, random_v: Option<Fr> (derived impl)

Container framing is ark-serialize's (un-vendored, restated): a Vec is a little-endian u64 length followed by the
elements; an Option is one byte (0 / 1) followed by the value; Fr is 32 little-endian canonical bytes.  The element work
(point encoding, decompression, on-curve and subgroup validation) runs on the GPU through pcgpu_g1_serialize /
pcgpu_g1_deserialize; this file only walks the framing.
"""
import struct

import numpy as np

from .binding import WireError  # noqa: F401  (re-exported: what deserialization raises)


def _vec_serialize(eng, curve, xy, inf, compressed):
    xy = np.asarray(xy, dtype=np.uint64)
    n = xy.reshape(-1, xy.shape[-1]).shape[0] if xy.size else 0
    body = eng.g1_serialize(curve, xy, inf, compressed).tobytes() if n else b""
    return struct.pack("<Q", n) + body


def _vec_deserialize(eng, curve, data, off, compressed, validate):
    if len(data) < off + 8:
        raise ValueError("truncated input (vector length)")
    (n,) = struct.unpack_from("<Q", data, off)
    off += 8
    sz = eng.g1_wire_size(curve, compressed)
    if len(data) < off + n * sz:
        raise ValueError("truncated input (vector body)")
    xy, inf = eng.g1_deserialize(curve, np.frombuffer(data, dtype=np.uint8, count=n * sz, offset=off), n, compressed, validate)
    return xy, inf, off + n * sz


def powers_serialize(eng, curve, powers_of_g, powers_of_gamma_g, compressed=True, inf_g=None, inf_gamma=None):
    """Powers::serialize_with_mode (data_structures.rs:142-156): the two vectors back to back."""
    return (_vec_serialize(eng, curve, powers_of_g, inf_g, compressed)
            + _vec_serialize(eng, curve, powers_of_gamma_g, inf_gamma, compressed))


def powers_deserialize(eng, curve, data, compressed=True, validate=True):
    """Powers::deserialize_with_mode (data_structures.rs:159-177) -> ((xy, inf) of powers_of_g, (xy, inf) of powers_of_gamma_g).
    Powers::check is a no-op (:137-141); element validation happens inside the vector reads, as in the reference."""
    data = bytes(data)
    g_xy, g_inf, off = _vec_deserialize(eng, curve, data, 0, compressed, validate)
    h_xy, h_inf, off = _vec_deserialize(eng, curve, data, off, compressed, validate)
    return (g_xy, g_inf), (h_xy, h_inf)


def commitment_serialize(eng, curve, comm_xy, comm_inf=False, compressed=True):
    """kzg10::Commitment(G1Affine), data_structures.rs:315-328"""
    inf = np.array([1 if comm_inf else 0], dtype=np.uint8)
    return eng.g1_serialize(curve, np.asarray(comm_xy, dtype=np.uint64).reshape(1, -1), inf, compressed).tobytes()


def commitment_deserialize(eng, curve, data, compressed=True, validate=True):
    xy, inf = eng.g1_deserialize(curve, bytes(data), 1, compressed, validate)
    return xy[0], bool(inf[0])


def proof_serialize(eng, curve, w_xy, w_inf=False, random_v=None, compressed=True):
    """kzg10::Proof { w, random_v: Option<Fr> }, data_structures.rs:479-495.  random_v: (4,) uint64 Montgomery or None."""
    out = commitment_serialize(eng, curve, w_xy, w_inf, compressed)
    if random_v is None:
        return out + b"\x00"
    canon = eng.fr_from_mont(curve, np.asarray(random_v, dtype=np.uint64).reshape(1, 4))
    return out + b"\x01" + canon.astype("<u8").tobytes()


def proof_deserialize(eng, curve, data, compressed=True, validate=True):
    """-> (w_xy, w_is_identity, random_v Montgomery (4,) uint64 or None)"""
    data = bytes(data)
    sz = eng.g1_wire_size(curve, compressed)
    w, winf = commitment_deserialize(eng, curve, data[:sz], compressed, validate)
    if len(data) < sz + 1 or data[sz] not in (0, 1):
        raise ValueError("malformed Option<Fr>")
    if data[sz] == 0:
        return w, winf, None
    from .params import FR_MODULUS, fr_mont
    v = int.from_bytes(data[sz + 1:sz + 33], "little")
    if len(data) < sz + 33 or v >= FR_MODULUS[curve]:
        raise ValueError("random_v is not a canonical field element")
    return w, winf, fr_mont(curve, v)


# ---- UniversalParams / VerifierKey (kzg10/data_structures.rs:22-112, :196-262) ---------------------------------------------
#   UniversalParams  powers_of_g: Vec<G1Affine> | powers_of_gamma_g: BTreeMap<usize, G1Affine> | h: G2Affine |
#                    beta_h: G2Affine | neg_powers_of_h: BTreeMap<usize, G2Affine>           (serialize_with_mode :61-74)
#   VerifierKey      g: G1Affine | gamma_g: G1Affine | h: G2Affine | beta_h: G2Affine          (:222-233)
# A BTreeMap is framed like a Vec of (key, value) pairs in ascending key order: u64 length, then per entry the usize key as a
# little-endian u64 followed by the value.  prepared_h / prepared_beta_h are not part of the encoding (recomputed, :95-96).
# The reference decodes every field with Validate::No first (:88-93, :243-246) and then, for Validate::Yes, runs one
# whole-struct check (:106-108, :41-48): a malformed ENCODING anywhere in the stream is reported before a validation failure
# of an earlier element.  `_Deferred` reproduces that precedence while still validating on the device in the same pass.
from . import g2_host  # noqa: E402


class _Deferred:
    """first validation-class failure seen so far (section, index, reason); encoding-class failures raise at once"""

    def __init__(self):
        self.first = None

    def note(self, section, index, reason):
        if self.first is None:
            self.first = (section, index, reason)


class KeyError_(ValueError):
    """SerializationError while reading a key: `section` names the field, `index` the element inside it"""

    def __init__(self, section, index, reason):
        super().__init__(f"{section}[{index}]: reason {reason}")
        self.section, self.index, self.reason = section, index, reason


def _g1_block(eng, curve, raw, n, compressed, validate, section, deferred):
    """n G1 elements (contiguous bytes) through the device decoder with the reference's error precedence"""
    if n == 0:
        nq = 2 * (6 if curve == 0 else 4)
        return np.zeros((0, nq), dtype=np.uint64), np.zeros(0, dtype=np.uint8)
    try:
        return eng.g1_deserialize(curve, raw, n, compressed, validate)
    except WireError as e:
        encoding = e.reason in (1, 2) or (e.reason == 3 and compressed)      # flags, non-canonical, x without a point
        if encoding or not validate:
            raise KeyError_(section, e.index, e.reason)
        deferred.note(section, e.index, e.reason)
        # a later element may still carry an ENCODING error, which takes precedence: decode again without validation
        try:
            return eng.g1_deserialize(curve, raw, n, compressed, False)
        except WireError as e2:
            raise KeyError_(section, e2.index, e2.reason)


def _map_g1_deserialize(eng, curve, data, off, compressed, validate, section, deferred):
    if len(data) < off + 8:
        raise ValueError("truncated input (map length)")
    (n,) = struct.unpack_from("<Q", data, off)
    off += 8
    sz = eng.g1_wire_size(curve, compressed)
    if len(data) < off + n * (8 + sz):
        raise ValueError("truncated input (map body)")
    rec = np.frombuffer(data, dtype=np.uint8, count=n * (8 + sz), offset=off).reshape(n, 8 + sz)
    keys = np.ascontiguousarray(rec[:, :8]).view("<u8").reshape(-1).astype(np.uint64)
    if n > 1 and not (keys[1:] > keys[:-1]).all():
        raise ValueError("BTreeMap keys are not strictly ascending")
    xy, inf = _g1_block(eng, curve, np.ascontiguousarray(rec[:, 8:]).reshape(-1), n, compressed, validate, section, deferred)
    return keys, xy, inf, off + n * (8 + sz)


def _map_g1_serialize(eng, curve, keys, xy, inf, compressed):
    keys = np.asarray(keys, dtype=np.uint64).reshape(-1)
    n = keys.size
    if n > 1 and not (keys[1:] > keys[:-1]).all():
        raise ValueError("keys must be strictly ascending (BTreeMap iteration order)")
    if n == 0:
        return struct.pack("<Q", 0)
    body = eng.g1_serialize(curve, np.asarray(xy, dtype=np.uint64).reshape(n, -1), inf, compressed)
    rec = np.concatenate([keys.astype("<u8").view(np.uint8).reshape(n, 8), body], axis=1)
    return struct.pack("<Q", n) + rec.tobytes()


def _g2_read(curve, data, off, compressed, validate, section, index, deferred):
    sz = g2_host.g2_wire_size(curve, compressed)
    if len(data) < off + sz:
        raise ValueError("truncated input (G2 element)")
    try:
        P = g2_host.g2_deserialize(curve, data[off:off + sz], compressed, validate=False)
    except g2_host.G2WireError as e:
        raise KeyError_(section, index, e.reason)
    if validate:
        try:
            g2_host.g2_check(curve, P)
        except g2_host.G2WireError as e:
            deferred.note(section, index, e.reason)
    return P, off + sz


def universal_params_serialize(eng, curve, powers_of_g, gamma_keys, gamma_xy, h, beta_h, neg_powers_of_h, compressed=True,
                               inf_g=None, inf_gamma=None):
    """UniversalParams::serialize_with_mode (data_structures.rs:61-74).  powers_of_g: (n, 2*limbs) Montgomery rows;
    gamma_keys / gamma_xy: the BTreeMap<usize, G1Affine> as ascending keys + rows; h, beta_h: G2 affine points
    ((x0, x1), (y0, y1)) or None; neg_powers_of_h: {key: G2 point}."""
    out = _vec_serialize(eng, curve, powers_of_g, inf_g, compressed)
    out += _map_g1_serialize(eng, curve, gamma_keys, gamma_xy, inf_gamma, compressed)
    out += g2_host.g2_serialize(curve, h, compressed) + g2_host.g2_serialize(curve, beta_h, compressed)
    out += struct.pack("<Q", len(neg_powers_of_h))
    for k in sorted(neg_powers_of_h):
        out += struct.pack("<Q", k) + g2_host.g2_serialize(curve, neg_powers_of_h[k], compressed)
    return out


def universal_params_deserialize(eng, curve, data, compressed=True, validate=True):
    """UniversalParams::deserialize_with_mode (data_structures.rs:83-111) -> dict(powers_of_g=(xy, inf), powers_of_gamma_g=
    (keys, xy, inf), h, beta_h, neg_powers_of_h={key: point}).  The G1 vectors (2^20+ points in a real SRS) are decompressed
    and validated on the GPU; raises KeyError_ naming the field and element like the reference's SerializationError."""
    data = bytes(data)
    d = _Deferred()
    if len(data) < 8:
        raise ValueError("truncated input (vector length)")
    (n,) = struct.unpack_from("<Q", data, 0)
    sz = eng.g1_wire_size(curve, compressed)
    if len(data) < 8 + n * sz:
        raise ValueError("truncated input (vector body)")
    g_xy, g_inf = _g1_block(eng, curve, np.frombuffer(data, dtype=np.uint8, count=n * sz, offset=8), n, compressed, validate, "powers_of_g", d)
    off = 8 + n * sz
    keys, gam_xy, gam_inf, off = _map_g1_deserialize(eng, curve, data, off, compressed, validate, "powers_of_gamma_g", d)
    h, off = _g2_read(curve, data, off, compressed, validate, "h", 0, d)
    beta_h, off = _g2_read(curve, data, off, compressed, validate, "beta_h", 0, d)
    if len(data) < off + 8:
        raise ValueError("truncated input (map length)")
    (m,) = struct.unpack_from("<Q", data, off)
    off += 8
    neg, last = {}, -1
    for i in range(m):
        if len(data) < off + 8:
            raise ValueError("truncated input (map key)")
        (k,) = struct.unpack_from("<Q", data, off)
        if k <= last and i:
            raise ValueError("BTreeMap keys are not strictly ascending")
        P, off = _g2_read(curve, data, off + 8, compressed, validate, "neg_powers_of_h", i, d)
        neg[k], last = P, k
    if d.first is not None:
        raise KeyError_(*d.first)
    return dict(powers_of_g=(g_xy, g_inf), powers_of_gamma_g=(keys, gam_xy, gam_inf), h=h, beta_h=beta_h, neg_powers_of_h=neg,
                consumed=off)


def verifier_key_serialize(eng, curve, g, gamma_g, h, beta_h, compressed=True):
    """VerifierKey::serialize_with_mode (data_structures.rs:222-233)"""
    pts = np.stack([np.asarray(g, dtype=np.uint64).reshape(-1), np.asarray(gamma_g, dtype=np.uint64).reshape(-1)])
    return (eng.g1_serialize(curve, pts, None, compressed).tobytes()
            + g2_host.g2_serialize(curve, h, compressed) + g2_host.g2_serialize(curve, beta_h, compressed))


def verifier_key_deserialize(eng, curve, data, compressed=True, validate=True):
    """VerifierKey::deserialize_with_mode (data_structures.rs:243-262) -> dict(g, gamma_g, h, beta_h)"""
    data = bytes(data)
    d = _Deferred()
    sz = eng.g1_wire_size(curve, compressed)
    if len(data) < 2 * sz:
        raise ValueError("truncated input")
    xy, inf = _g1_block(eng, curve, np.frombuffer(data, dtype=np.uint8, count=2 * sz), 2, compressed, validate, "g/gamma_g", d)
    h, off = _g2_read(curve, data, 2 * sz, compressed, validate, "h", 0, d)
    beta_h, off = _g2_read(curve, data, off, compressed, validate, "beta_h", 0, d)
    if d.first is not None:
        raise KeyError_(*d.first)
    return dict(g=(xy[0], bool(inf[0])), gamma_g=(xy[1], bool(inf[1])), h=h, beta_h=beta_h, consumed=off)


def sonic_verifier_key_serialize(eng, curve, g, gamma_g, h, beta_h, degree_bounds_and_neg_powers_of_h, supported_degree, max_degree,
                                 compressed=True):
    """SonicKZG10 VerifierKey::serialize_with_mode (sonic_pc/data_structures.rs:190-216): g, gamma_g, h, beta_h, then
    Option<Vec<(usize, G2Affine)>> (a 1-byte tag, a u64 length, each bound as u64 and its point), supported_degree, max_degree"""
    out = verifier_key_serialize(eng, curve, g, gamma_g, h, beta_h, compressed)
    if degree_bounds_and_neg_powers_of_h is None:
        out += b"\x00"
    else:
        out += b"\x01" + struct.pack("<Q", len(degree_bounds_and_neg_powers_of_h))
        for bound, P in degree_bounds_and_neg_powers_of_h:
            out += struct.pack("<Q", bound) + g2_host.g2_serialize(curve, P, compressed)
    return out + struct.pack("<QQ", supported_degree, max_degree)


def sonic_verifier_key_deserialize(eng, curve, data, compressed=True, validate=True):
    """SonicKZG10 VerifierKey::deserialize_with_mode (sonic_pc/data_structures.rs:218-262) -> dict(g, gamma_g, h, beta_h,
    degree_bounds_and_neg_powers_of_h=None or [(bound, point)], supported_degree, max_degree); Valid::check's
    supported_degree > max_degree is InvalidData (:153-155)"""
    data = bytes(data)
    d = _Deferred()
    sz = eng.g1_wire_size(curve, compressed)
    if len(data) < 2 * sz:
        raise ValueError("truncated input")
    xy, inf = _g1_block(eng, curve, np.frombuffer(data, dtype=np.uint8, count=2 * sz), 2, compressed, validate, "g/gamma_g", d)
    h, off = _g2_read(curve, data, 2 * sz, compressed, validate, "h", 0, d)
    beta_h, off = _g2_read(curve, data, off, compressed, validate, "beta_h", 0, d)
    if len(data) < off + 1:
        raise ValueError("truncated input (option tag)")
    tag, off = data[off], off + 1
    if tag > 1:
        raise ValueError("invalid option tag")
    bounds = None
    if tag:
        if len(data) < off + 8:
            raise ValueError("truncated input (vector length)")
        (m,) = struct.unpack_from("<Q", data, off)
        off += 8
        bounds = []
        for i in range(m):
            if len(data) < off + 8:
                raise ValueError("truncated input (degree bound)")
            (b,) = struct.unpack_from("<Q", data, off)
            P, off = _g2_read(curve, data, off + 8, compressed, validate, "degree_bounds_and_neg_powers_of_h", i, d)
            bounds.append((b, P))
    if len(data) < off + 16:
        raise ValueError("truncated input (degrees)")
    supported_degree, max_degree = struct.unpack_from("<QQ", data, off)
    if d.first is not None:
        raise KeyError_(*d.first)
    if validate and supported_degree > max_degree:
        raise ValueError("InvalidData: supported_degree > max_degree")
    return dict(g=(xy[0], bool(inf[0])), gamma_g=(xy[1], bool(inf[1])), h=h, beta_h=beta_h,
                degree_bounds_and_neg_powers_of_h=bounds, supported_degree=supported_degree, max_degree=max_degree,
                consumed=off + 16)


# ---- BrakedownPCParams (linear_codes/data_structures.rs:12-61), derived CanonicalSerialize -------------------------------
# Field order of the struct; usize = u64 LE, Vec = u64 length + elements, tuples element by element, SprsMat = n, m, d,
# ind_ptr, col_ind, val (linear_codes/utils.rs:20-37), Fr = 32 canonical LE bytes, bool = one byte.  The three hash
# parameters are `()` in the configuration of the reference's tests and benches and contribute no bytes.  Needs no device.
def _fr_canon_bytes(curve, val):
    from .params import FR_MODULUS
    r = FR_MODULUS[curve]
    rinv = pow(1 << 256, -1, r)
    out = bytearray()
    for x in np.asarray(val, dtype=np.uint64).reshape(-1, 4):
        v = (int(x[0]) | int(x[1]) << 64 | int(x[2]) << 128 | int(x[3]) << 192) * rinv % r
        out += v.to_bytes(32, "little")
    return bytes(out)


def brakedown_params_serialize(params):
    curve = params["curve"]
    q = lambda *v: struct.pack("<%dQ" % len(v), *v)
    vec = lambda xs: q(len(xs)) + b"".join(q(*x) if isinstance(x, tuple) else q(x) for x in xs)
    out = bytearray(q(params["sec_param"], *params["alpha"], *params["beta"], *params["rho_inv"], params["base_len"], params["n"],
                      params["m"], params["m_ext"]))
    out += vec([tuple(x) for x in params["a_dims"]]) + vec([tuple(x) for x in params["b_dims"]])
    out += vec(list(params["start"])) + vec(list(params["end"]))
    for mats, dims in ((params["a_mats"], params["a_dims"]), (params["b_mats"], params["b_dims"])):
        out += q(len(mats))
        for (ind_ptr, col_ind, val), (n, m, d) in zip(mats, dims):
            out += q(n, m, d) + vec([int(x) for x in ind_ptr]) + vec([int(x) for x in col_ind])
            out += q(len(val)) + _fr_canon_bytes(curve, val)
    out += bytes([1 if params["check_well_formedness"] else 0])
    return bytes(out)


def brakedown_params_deserialize(curve, data):
    """inverse of brakedown_params_serialize; ValueError on a truncated buffer, trailing bytes, a bool other than 0 / 1 or a
    field element >= r"""
    from .params import FR_MODULUS, fr_mont
    r = FR_MODULUS[curve]
    data = bytes(data)
    pos = [0]

    def take(n):
        if pos[0] + n > len(data):
            raise ValueError("truncated BrakedownPCParams")
        b = data[pos[0]:pos[0] + n]
        pos[0] += n
        return b

    u = lambda: struct.unpack("<Q", take(8))[0]
    vec = lambda k: [tuple(u() for _ in range(k)) if k > 1 else u() for _ in range(u())]
    p = dict(curve=curve, sec_param=u(), alpha=(u(), u()), beta=(u(), u()), rho_inv=(u(), u()), base_len=u(), n=u(), m=u(), m_ext=u())
    p["a_dims"], p["b_dims"] = vec(3), vec(3)
    p["start"], p["end"] = vec(1), vec(1)
    for key in ("a_mats", "b_mats"):
        mats = []
        for _ in range(u()):
            u(), u(), u()                               # n, m, d: repeated from the dims
            ind_ptr = np.array(vec(1), dtype=np.uint64)
            col_ind = np.array(vec(1), dtype=np.uint64)
            vals = []
            for _ in range(u()):
                v = int.from_bytes(take(32), "little")
                if v >= r:
                    raise ValueError("field element out of range")
                vals.append(fr_mont(curve, v))
            mats.append((ind_ptr, col_ind, np.array(vals, dtype=np.uint64).reshape(-1, 4)))
        p[key] = mats
    flag = take(1)[0]
    if flag > 1:
        raise ValueError("invalid bool")
    p["check_well_formedness"] = bool(flag)
    if pos[0] != len(data):
        raise ValueError("trailing bytes after BrakedownPCParams")
    return p
