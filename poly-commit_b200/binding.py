"""ctypes binding of include/pcgpu.h.  Arrays are numpy uint64 in the ABI's packed layout
(little-endian limbs; Montgomery unless stated) or raw device pointers (ints) with DEVICE_PTRS."""
import ctypes
import os

import numpy as np

BLS12_381, BN254, PALLAS = 0, 1, 2
CURVES = {"bls12_381": BLS12_381, "bn254": BN254, "pallas": PALLAS}
# pcgpu_msm_last_geometry: field names in the header's PCGPU_GEOM_* order, and the PCGPU_MSM_PATH_* values
GEOM_FIELDS = ("path", "split", "n", "c", "W", "G", "R", "T", "tdiv", "wave", "entries", "heavy")
MSM_PATH_NONE, MSM_PATH_SMALL, MSM_PATH_BUCKETS = 0, 1, 2
SCALARS_MONT, DEVICE_PTRS, SRS_PRECOMPUTE, NTT_INVERSE, SRS_COMB, WIRE_COMPRESSED, WIRE_NO_VALIDATE = 1, 2, 4, 8, 16, 32, 64
E_INVALID = -8

_HERE = os.path.dirname(os.path.abspath(__file__))


def fq_limbs(curve):
    return 6 if curve == BLS12_381 else 4


def library_path():
    return os.path.join(_HERE, "libpcgpu.so")


class PcgpuError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"pcgpu error {code}: {msg}")
        self.code = code


class WireError(PcgpuError):
    """SerializationError from g1_deserialize: `index` of the first offending element and `reason`
    (1 unexpected flags, 2 coordinate >= p, 3 not on the curve, 4 not in the prime-order subgroup)."""

    def __init__(self, code, msg, index, reason):
        super().__init__(code, f"{msg} (element {index}, reason {reason})")
        self.index, self.reason = index, reason


_sz = ctypes.c_size_t
_vp = ctypes.c_void_p


def _load(path):
    if not os.path.exists(path):
        raise ImportError(
            f"{path} not found: the CUDA library is required (build it with `python -c 'import __graft_entry__ as g; "
            f"g.build()'`); there is no CPU fallback")
    lib = ctypes.CDLL(path)
    lib.pcgpu_strerror.restype = ctypes.c_char_p
    lib.pcgpu_strerror.argtypes = [ctypes.c_int]
    lib.pcgpu_srs_len.restype = _sz
    lib.pcgpu_srs_len.argtypes = [_vp]
    lib.pcgpu_srs_curve.argtypes = [_vp]
    lib.pcgpu_ipa_len.restype = _sz
    lib.pcgpu_ipa_len.argtypes = [_vp]
    lib.pcgpu_g1_wire_size.restype = _sz
    lib.pcgpu_g1_wire_size.argtypes = [ctypes.c_int, ctypes.c_uint32]
    lib.pcgpu_launch_count.restype = ctypes.c_uint64
    lib.pcgpu_launch_count.argtypes = []
    lib.pcgpu_peer_window_bytes.restype = _sz
    lib.pcgpu_peer_window_bytes.argtypes = []
    sigs = {
        "pcgpu_init": [ctypes.c_int, ctypes.POINTER(_vp)],
        "pcgpu_destroy": [_vp],
        "pcgpu_set_stream": [_vp, _vp],
        "pcgpu_profile_enable": [_vp, ctypes.c_int],
        "pcgpu_profile_get": [_vp, ctypes.c_int, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_uint64)],
        "pcgpu_srs_register": [_vp, ctypes.c_int, _vp, _vp, _sz, ctypes.c_uint32, ctypes.POINTER(_vp)],
        "pcgpu_srs_release": [_vp, _vp],
        "pcgpu_msm": [_vp, _vp, _sz, _vp, _sz, ctypes.c_uint32, _vp, _vp],
        "pcgpu_msm_batch": [_vp, _vp, _vp, _sz, _sz, ctypes.c_uint32, _vp, _vp],
        "pcgpu_msm_partial": [_vp, _vp, _sz, _vp, _sz, ctypes.c_uint32, _vp],
        "pcgpu_g1_sum_xyzz": [_vp, ctypes.c_int, _vp, _sz, _vp, _vp],
        "pcgpu_g1_fixed_base_mul": [_vp, ctypes.c_int, _vp, _vp, _sz, ctypes.c_uint32, _vp],
        "pcgpu_fr_from_mont": [_vp, ctypes.c_int, _vp, _vp, _sz, ctypes.c_uint32],
        "pcgpu_fr_mul": [_vp, ctypes.c_int, _vp, _vp, _vp, _sz, ctypes.c_uint32],
        "pcgpu_msm_bases": [_vp, ctypes.c_int, _vp, _vp, _vp, _sz, ctypes.c_uint32, _vp, _vp],
        "pcgpu_fr_axpy": [_vp, ctypes.c_int, _vp, _vp, _vp, _sz, ctypes.c_uint32],
        "pcgpu_fr_div_linear": [_vp, ctypes.c_int, _vp, _sz, _vp, _vp, _vp, ctypes.c_uint32],
        "pcgpu_fr_inner_product": [_vp, ctypes.c_int, _vp, _vp, _sz, _vp, ctypes.c_uint32],
        "pcgpu_fr_row_mul": [_vp, ctypes.c_int, _vp, _vp, _sz, _sz, _vp, ctypes.c_uint32],
        "pcgpu_measure_imad_peak": [_vp, ctypes.POINTER(ctypes.c_double)],
        "pcgpu_selftest_field": [_vp, ctypes.c_int, ctypes.c_uint64, _sz, ctypes.POINTER(ctypes.c_uint64)],
        "pcgpu_msm_last_geometry": [_vp, ctypes.POINTER(ctypes.c_uint64), _sz],
        "pcgpu_diag_field_op": [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp, _sz],
        "pcgpu_ipa_begin": [_vp, ctypes.c_int, _vp, _sz, _vp, _sz, _vp, ctypes.c_uint32, ctypes.POINTER(_vp)],
        "pcgpu_ipa_round_lr": [_vp, _vp, _vp, _vp, _vp, _vp, _vp],
        "pcgpu_ipa_round_fold": [_vp, _vp, _vp, _vp],
        "pcgpu_ipa_check_final_key": [_vp, _vp, _vp, ctypes.c_uint32, _vp, _vp],
        "pcgpu_ipa_finish": [_vp, _vp, _vp, _vp],
        "pcgpu_g1_serialize": [_vp, ctypes.c_int, _vp, _vp, _sz, ctypes.c_uint32, _vp],
        "pcgpu_g1_deserialize": [_vp, ctypes.c_int, _vp, _sz, ctypes.c_uint32, _vp, _vp, ctypes.POINTER(_sz),
                                 ctypes.POINTER(ctypes.c_int)],
        "pcgpu_ntt_split": [ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint32)],
        "pcgpu_ntt_pass": [_vp, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_int, _sz, _sz, _vp, _sz, _vp],
        "pcgpu_ntt_pass1_peer": [_vp, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32, _sz, _sz, _vp, _sz, ctypes.POINTER(_vp),
                                 ctypes.c_uint32],
        "pcgpu_ntt_batch": [_vp, ctypes.c_int, _vp, _sz, _sz, ctypes.c_uint32, ctypes.c_uint32, _vp],
        "pcgpu_ntt": [_vp, ctypes.c_int, _vp, _sz, ctypes.c_uint32, ctypes.c_uint32, _vp],
        "pcgpu_kzg_commit_batch": [_vp, _vp, _vp, _vp, _sz, ctypes.c_uint32, _vp, _vp],
        "pcgpu_kzg_commit": [_vp, _vp, _vp, _sz, _vp, _vp, _sz, ctypes.c_uint32, _vp, _vp],
        "pcgpu_kzg_open": [_vp, _vp, _vp, _sz, _vp, _vp, _vp, _sz, ctypes.c_uint32, _vp, _vp, _vp],
        "pcgpu_g1_sample_generators": [_vp, ctypes.c_int, _vp, _sz, ctypes.c_uint64, _sz, ctypes.c_uint32, _vp],
        "pcgpu_buf_alloc": [_vp, _sz, ctypes.POINTER(_vp)],
        "pcgpu_buf_free": [_vp, _vp],
        "pcgpu_buf_write": [_vp, _vp, _sz, _vp, _sz],
        "pcgpu_buf_read": [_vp, _vp, _sz, _vp, _sz],
        "pcgpu_buf_zero": [_vp, _vp, _sz, _sz],
        "pcgpu_kzg_commit_open": [_vp, _vp, _vp, _sz, _vp, ctypes.c_uint32, _vp, _vp, _vp, _vp],
        "pcgpu_kzg_commit_open_batch": [_vp, _vp, _vp, _vp, _sz, _vp, ctypes.c_uint32, _vp, _vp, _vp, _vp],
        "pcgpu_lincode_hash_columns": [_vp, ctypes.c_int, _vp, _sz, _sz, ctypes.c_int, ctypes.c_uint32, _vp],
        "pcgpu_merkle_tree": [_vp, _vp, _sz, ctypes.c_uint32, _vp, _vp],
        "pcgpu_lincode_commit": [_vp, ctypes.c_int, _vp, _sz, _sz, ctypes.c_uint32, ctypes.c_int, ctypes.c_uint32, _vp, _vp, _vp, _vp],
        "pcgpu_peer_alloc": [_vp, _sz, ctypes.POINTER(_vp), _vp],
        "pcgpu_peer_open": [_vp, _vp, ctypes.POINTER(_vp)],
        "pcgpu_peer_close": [_vp, _vp],
        "pcgpu_peer_free": [_vp, _vp],
        "pcgpu_peer_signal": [_vp, ctypes.POINTER(_vp), ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64],
        "pcgpu_peer_wait": [_vp, _vp, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64],
        "pcgpu_msm_peer": [_vp, _vp, _sz, _vp, _sz, ctypes.c_uint32, ctypes.POINTER(_vp), ctypes.c_uint32, ctypes.c_uint32,
                           ctypes.c_uint64, _vp, _vp],
    }
    for name, args in sigs.items():
        fn = getattr(lib, name, None)
        if fn is None:      # a library older than this binding: only the calls that need the symbol fail (AttributeError)
            continue
        fn.argtypes = args
        fn.restype = None if name in ("pcgpu_destroy", "pcgpu_srs_release") else ctypes.c_int
    return lib


def _ptr(a):
    """numpy array -> pointer; int -> device pointer; None -> NULL."""
    if a is None:
        return None
    if isinstance(a, (int, np.integer)):
        return ctypes.c_void_p(int(a))
    return a.ctypes.data_as(ctypes.c_void_p)


def _u64(a):
    if a is None or isinstance(a, (int, np.integer)):
        return a
    return np.ascontiguousarray(a, dtype=np.uint64)


class Srs:
    """Device-resident bases (kzg10 Powers::powers_of_g / powers_of_gamma_g, ipa comm_key, hyrax com_key)."""

    def __init__(self, engine, handle, curve, n):
        self.engine, self.handle, self.curve, self.n = engine, handle, curve, n

    def __len__(self):
        return self.n

    def release(self):
        if self.handle is not None:
            self.engine.lib.pcgpu_srs_release(self.engine.ctx, self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class DeviceBuffer:
    """`count` Fr elements (32 bytes each) on the engine's device; `ptr(i)` is the device pointer of element i, to be passed
    with DEVICE_PTRS.  Freed on release() / garbage collection."""

    def __init__(self, engine, count):
        self.engine, self.count = engine, count
        p = _vp()
        engine._ck(engine.lib.pcgpu_buf_alloc(engine.ctx, max(count, 1) * 32, ctypes.byref(p)))
        self.base = int(p.value)

    def ptr(self, i=0):
        return self.base + 32 * i

    def write(self, arr, at=0):
        arr = np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1, 4)
        if at + arr.shape[0] > self.count:
            raise ValueError("write beyond the buffer")
        self.engine._ck(self.engine.lib.pcgpu_buf_write(self.engine.ctx, _vp(self.base), 32 * at, _ptr(arr), arr.shape[0] * 32))

    def read(self, at=0, count=None):
        count = self.count - at if count is None else count
        out = np.zeros((count, 4), dtype=np.uint64)
        self.engine._ck(self.engine.lib.pcgpu_buf_read(self.engine.ctx, _vp(self.base), 32 * at, _ptr(out), count * 32))
        return out

    def zero(self, at=0, count=None):
        count = self.count - at if count is None else count
        self.engine._ck(self.engine.lib.pcgpu_buf_zero(self.engine.ctx, _vp(self.base), 32 * at, count * 32))

    def release(self):
        if getattr(self, "base", None) and getattr(self.engine, "ctx", None):
            b, self.base = self.base, None
            self.engine.lib.pcgpu_buf_free(self.engine.ctx, _vp(b))

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class IpaState:
    """Device-resident state of one InnerProductArgPC::open halving loop; released by ipa_finish, by release() or when the
    object is dropped (an exception between ipa_begin and ipa_finish therefore does not leak device memory)."""

    def __init__(self, engine, handle, curve):
        self.engine, self.handle, self.curve = engine, handle, curve

    def release(self):
        if self.handle is not None and getattr(self.engine, "ctx", None):
            h, self.handle = self.handle, None
            self.engine.lib.pcgpu_ipa_finish(self.engine.ctx, h, None, None)

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class Engine:
    """One pcgpu context (one CUDA device, one stream).  `lib_path` exists so the host-emulation unit tests
    can drive the identical C ABI of tests/host_emul/libpcgpu_hostcheck.so; product code never passes it."""

    def __init__(self, device=0, lib_path=None):
        self.lib = _load(lib_path or library_path())
        ctx = _vp()
        rc = self.lib.pcgpu_init(device, ctypes.byref(ctx))
        if rc:
            raise PcgpuError(rc, self.lib.pcgpu_strerror(rc).decode())
        self.ctx = ctx
        self.device = device

    def close(self):
        if getattr(self, "ctx", None):
            self.lib.pcgpu_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc:
            raise PcgpuError(rc, self.lib.pcgpu_strerror(rc).decode())

    def buffer(self, count):
        """zero-filled device buffer of `count` Fr elements"""
        return DeviceBuffer(self, count)

    # ---- context ----
    def set_stream(self, cuda_stream):
        self._ck(self.lib.pcgpu_set_stream(self.ctx, _vp(cuda_stream) if cuda_stream else None))

    def profile_enable(self, on=True):
        self._ck(self.lib.pcgpu_profile_enable(self.ctx, 1 if on else 0))

    def profile_get(self, stage):
        ms, cnt = ctypes.c_double(), ctypes.c_uint64()
        self._ck(self.lib.pcgpu_profile_get(self.ctx, stage, ctypes.byref(ms), ctypes.byref(cnt)))
        return ms.value, cnt.value

    def launch_count(self):
        return int(self.lib.pcgpu_launch_count())

    def measure_imad_peak(self):
        v = ctypes.c_double()
        self._ck(self.lib.pcgpu_measure_imad_peak(self.ctx, ctypes.byref(v)))
        return v.value

    def selftest_field(self, curve, seed=1, n=4096):
        bad = ctypes.c_uint64()
        self._ck(self.lib.pcgpu_selftest_field(self.ctx, curve, seed, n, ctypes.byref(bad)))
        return bad.value

    def msm_last_geometry(self):
        """dict of the path and geometry the most recent MSM on this context took (pcgpu_msm_last_geometry; keys GEOM_FIELDS;
        "heavy" is None where the pipeline did not report it)."""
        out = (ctypes.c_uint64 * len(GEOM_FIELDS))()
        self._ck(self.lib.pcgpu_msm_last_geometry(self.ctx, out, len(GEOM_FIELDS)))
        g = dict(zip(GEOM_FIELDS, (int(v) for v in out)))
        if g["heavy"] == 2**64 - 1:
            g["heavy"] = None
        return g

    def diag_field_op(self, curve, which, op, a, b):
        """one field primitive elementwise on the device (pcgpu_diag_field_op): which 0 = Fq, 1 = Fr of `curve`; a, b: (n, limbs)
        uint64 Montgomery elements (limbs = 6 for BLS12-381 Fq, else 4); returns the (n, limbs) results."""
        a, b = _u64(a), _u64(b)
        if a.shape != b.shape:
            raise ValueError("operand shapes differ")
        out = np.zeros_like(a)
        self._ck(self.lib.pcgpu_diag_field_op(self.ctx, curve, which, op, _ptr(a), _ptr(b), _ptr(out), a.shape[0]))
        return out

    # ---- SRS ----
    def srs_register(self, curve, bases_xy, inf=None, n=None, flags=0):
        bases_xy = _u64(bases_xy)
        if n is None:
            n = bases_xy.size // (2 * fq_limbs(curve))
        inf = None if inf is None else np.ascontiguousarray(inf, dtype=np.uint8)
        h = _vp()
        self._ck(self.lib.pcgpu_srs_register(self.ctx, curve, _ptr(bases_xy), _ptr(inf), n, flags, ctypes.byref(h)))
        return Srs(self, h, curve, n)

    # ---- MSM ----
    def msm(self, srs, scalars, n=None, base_offset=0, flags=0):
        """msm_bigint(&bases[base_offset..], scalars) -> (xy uint64[2*limbs], is_identity)."""
        scalars = _u64(scalars)
        if n is None:
            n = scalars.size // 4
        out = np.zeros(2 * fq_limbs(srs.curve), dtype=np.uint64)
        inf = np.zeros(1, dtype=np.uint8)
        self._ck(self.lib.pcgpu_msm(self.ctx, srs.handle, base_offset, _ptr(scalars), n, flags, _ptr(out), _ptr(inf)))
        return out, int(inf[0])

    def msm_batch(self, srs, scalars, n, count, flags=0):
        """count MSMs of length n over the same bases -> ((count, 2*limbs) uint64, (count,) uint8 identity flags)."""
        scalars = _u64(scalars)
        out = np.zeros((count, 2 * fq_limbs(srs.curve)), dtype=np.uint64)
        inf = np.zeros(count, dtype=np.uint8)
        self._ck(self.lib.pcgpu_msm_batch(self.ctx, srs.handle, _ptr(scalars), n, count, flags, _ptr(out), _ptr(inf)))
        return out, inf

    def msm_partial(self, srs, scalars, n=None, base_offset=0, flags=0):
        scalars = _u64(scalars)
        if n is None:
            n = scalars.size // 4
        out = np.zeros(4 * fq_limbs(srs.curve), dtype=np.uint64)
        self._ck(self.lib.pcgpu_msm_partial(self.ctx, srs.handle, base_offset, _ptr(scalars), n, flags, _ptr(out)))
        return out

    def g1_sum_xyzz(self, curve, xyzz):
        xyzz = _u64(xyzz)
        count = xyzz.size // (4 * fq_limbs(curve))
        out = np.zeros(2 * fq_limbs(curve), dtype=np.uint64)
        inf = np.zeros(1, dtype=np.uint8)
        self._ck(self.lib.pcgpu_g1_sum_xyzz(self.ctx, curve, _ptr(xyzz), count, _ptr(out), _ptr(inf)))
        return out, int(inf[0])

    def fixed_base_mul(self, curve, base_xy, scalars, n=None, flags=0, out=None):
        base_xy, scalars = _u64(base_xy), _u64(scalars)
        if n is None:
            n = scalars.size // 4
        if out is None:
            out = np.zeros((n, 2 * fq_limbs(curve)), dtype=np.uint64)
        self._ck(self.lib.pcgpu_g1_fixed_base_mul(self.ctx, curve, _ptr(base_xy), _ptr(scalars), n, flags, _ptr(out)))
        return out

    def g1_sample_generators(self, curve, protocol_name, n, first_index=0, flags=0, out=None):
        """InnerProductArgPC::sample_generators / HyraxPC::setup: n hash-derived points -> (n, 2*limbs) uint64"""
        name = np.frombuffer(bytes(protocol_name), dtype=np.uint8).copy()
        if out is None:
            out = np.zeros((n, 2 * fq_limbs(curve)), dtype=np.uint64)
        self._ck(self.lib.pcgpu_g1_sample_generators(self.ctx, curve, _ptr(name), name.size, first_index, n, flags, _ptr(out)))
        return out

    # ---- Fr ----
    def fr_mul(self, curve, a, b):
        """elementwise Montgomery product of two (n, 4) arrays"""
        a, b = _u64(a), _u64(b)
        n = a.size // 4
        out = np.zeros((n, 4), dtype=np.uint64)
        self._ck(self.lib.pcgpu_fr_mul(self.ctx, curve, _ptr(a), _ptr(b), _ptr(out), n, 0))
        return out

    def msm_bases(self, curve, bases_xy, scalars, inf=None, flags=0):
        """VariableBaseMSM::msm_bigint on unregistered bases -> (xy, is_identity)"""
        bases_xy, scalars = _u64(bases_xy), _u64(scalars)
        n = scalars.size // 4
        if bases_xy.size // (2 * fq_limbs(curve)) < n:
            raise ValueError("fewer bases than scalars")
        inf = None if inf is None else np.ascontiguousarray(inf, dtype=np.uint8)
        out = np.zeros(2 * fq_limbs(curve), dtype=np.uint64)
        oinf = np.zeros(1, dtype=np.uint8)
        self._ck(self.lib.pcgpu_msm_bases(self.ctx, curve, _ptr(bases_xy), _ptr(inf), _ptr(scalars), n, flags, _ptr(out), _ptr(oinf)))
        return out, bool(oinf[0])

    def fr_from_mont(self, curve, a, n=None, flags=0, out=None):
        a = _u64(a)
        if n is None:
            n = a.size // 4
        if out is None:
            out = np.zeros((n, 4), dtype=np.uint64)
        self._ck(self.lib.pcgpu_fr_from_mont(self.ctx, curve, _ptr(a), _ptr(out), n, flags))
        return out

    def fr_axpy(self, curve, y, c, x, n=None, flags=0):
        """y += c * x (in place when y is a device pointer; returns the updated host copy otherwise)."""
        c, x = _u64(c), _u64(x)
        if not isinstance(y, (int, np.integer)):
            y = _u64(y).copy()
        if n is None:
            n = x.size // 4
        self._ck(self.lib.pcgpu_fr_axpy(self.ctx, curve, _ptr(y), _ptr(c), _ptr(x), n, flags))
        return y

    def fr_div_linear(self, curve, p, z, n=None, flags=0, q=None):
        p, z = _u64(p), _u64(z)
        if n is None:
            n = p.size // 4
        if q is None:
            q = np.zeros((max(n - 1, 0), 4), dtype=np.uint64)
        rem = np.zeros(4, dtype=np.uint64)
        self._ck(self.lib.pcgpu_fr_div_linear(self.ctx, curve, _ptr(p), n, _ptr(z), _ptr(q), _ptr(rem), flags))
        return q, rem

    def fr_inner_product(self, curve, a, b, n=None, flags=0):
        a, b = _u64(a), _u64(b)
        if n is None:
            n = a.size // 4
        out = np.zeros(4, dtype=np.uint64)
        self._ck(self.lib.pcgpu_fr_inner_product(self.ctx, curve, _ptr(a), _ptr(b), n, _ptr(out), flags))
        return out

    def fr_row_mul(self, curve, v, m, rows, cols, flags=0):
        v, m = _u64(v), _u64(m)
        out = np.zeros((cols, 4), dtype=np.uint64)
        self._ck(self.lib.pcgpu_fr_row_mul(self.ctx, curve, _ptr(v), _ptr(m), rows, cols, _ptr(out), flags))
        return out

    def ntt(self, curve, coeffs, logn, n_in=None, inverse=False, flags=0, out=None):
        """EvaluationDomain::fft (zero-padded, natural order) / ifft."""
        coeffs = _u64(coeffs)
        if n_in is None:
            n_in = coeffs.size // 4
        if out is None:
            out = np.zeros((1 << logn, 4), dtype=np.uint64)
        self._ck(self.lib.pcgpu_ntt(self.ctx, curve, _ptr(coeffs), n_in, logn, flags | (NTT_INVERSE if inverse else 0), _ptr(out)))
        return out

    # ---- G1 wire formats (ark-serialize CanonicalSerialize / CanonicalDeserialize of G1Affine) ----
    def g1_wire_size(self, curve, compressed=True):
        return int(self.lib.pcgpu_g1_wire_size(curve, WIRE_COMPRESSED if compressed else 0))

    def g1_serialize(self, curve, xy, inf=None, compressed=True):
        """n affine points (Montgomery x||y, optional infinity bytes) -> (n, wire_size) uint8"""
        xy = _u64(xy)
        n = xy.size // (2 * fq_limbs(curve))
        inf = None if inf is None else np.ascontiguousarray(inf, dtype=np.uint8)
        out = np.zeros((n, self.g1_wire_size(curve, compressed)), dtype=np.uint8)
        self._ck(self.lib.pcgpu_g1_serialize(self.ctx, curve, _ptr(xy), _ptr(inf), n, WIRE_COMPRESSED if compressed else 0, _ptr(out)))
        return out

    def g1_deserialize(self, curve, data, n=None, compressed=True, validate=True):
        """bytes -> ((n, 2*limbs) uint64 Montgomery x||y, (n,) uint8 infinity); raises WireError like SerializationError"""
        data = np.ascontiguousarray(np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else data,
                                    dtype=np.uint8).reshape(-1)
        sz = self.g1_wire_size(curve, compressed)
        if n is None:
            n = data.size // sz
        if data.size < n * sz:
            raise ValueError("byte buffer shorter than n elements")
        xy = np.zeros((n, 2 * fq_limbs(curve)), dtype=np.uint64)
        inf = np.zeros(n, dtype=np.uint8)
        bad, reason = _sz(0), ctypes.c_int(0)
        flags = (WIRE_COMPRESSED if compressed else 0) | (0 if validate else WIRE_NO_VALIDATE)
        rc = self.lib.pcgpu_g1_deserialize(self.ctx, curve, _ptr(data), n, flags, _ptr(xy), _ptr(inf), ctypes.byref(bad),
                                           ctypes.byref(reason))
        if rc == E_INVALID:
            raise WireError(rc, self.lib.pcgpu_strerror(rc).decode(), int(bad.value), int(reason.value))
        self._ck(rc)
        return xy, inf

    def ntt_pass1_peer(self, curve, logn, lo, count, in_ptr, n_in, dst_ptrs, inverse=False):
        """pass 1 on columns [lo, lo+count) storing straight into the row buffers dst_ptrs[rank] (device pointers as ints)"""
        arr = (_vp * len(dst_ptrs))(*[ctypes.c_void_p(int(p)) for p in dst_ptrs])
        self._ck(self.lib.pcgpu_ntt_pass1_peer(self.ctx, curve, logn, NTT_INVERSE if inverse else 0, lo, count, _ptr(in_ptr), n_in, arr,
                                               len(dst_ptrs)))

    def ntt_batch(self, curve, rows, logn, inverse=False):
        """(count, n_in, 4) rows -> (count, 2^logn, 4): every row zero-padded and transformed (Ligero row encoding)"""
        rows = _u64(rows)
        count, n_in = rows.shape[0], rows.shape[1]
        out = np.zeros((count, 1 << logn, 4), dtype=np.uint64)
        self._ck(self.lib.pcgpu_ntt_batch(self.ctx, curve, _ptr(rows), n_in, count, logn, NTT_INVERSE if inverse else 0, _ptr(out)))
        return out

    def ntt_split(self, logn):
        m1, m2 = ctypes.c_uint32(), ctypes.c_uint32()
        self._ck(self.lib.pcgpu_ntt_split(logn, ctypes.byref(m1), ctypes.byref(m2)))
        return m1.value, m2.value

    def ntt_pass(self, curve, logn, which, lo, count, in_ptr, n_in, out_ptr, inverse=False):
        """one four-step pass on a slice of its batches; in_ptr / out_ptr are DEVICE pointers (ints)"""
        self._ck(self.lib.pcgpu_ntt_pass(self.ctx, curve, logn, NTT_INVERSE if inverse else 0, which, lo, count, _ptr(in_ptr), n_in,
                                         _ptr(out_ptr)))

    # ---- linear-code commitments: column hashes + Merkle tree ----
    def lincode_hash_columns(self, curve, ext_mat, n_rows=None, n_cols=None, hash=0, flags=0, out=None):
        """leaves[j] = D(to_bytes!(column j)) for a row-major (n_rows, n_cols, 4) Montgomery matrix -> (n_cols, 32) uint8"""
        ext_mat = _u64(ext_mat)
        if n_rows is None:
            n_rows, n_cols = ext_mat.shape[0], ext_mat.shape[1]
        if out is None:
            out = np.zeros((n_cols, 32), dtype=np.uint8)
        self._ck(self.lib.pcgpu_lincode_hash_columns(self.ctx, curve, _ptr(ext_mat), n_rows, n_cols, hash, flags, _ptr(out)))
        return out

    def merkle_tree(self, leaves, n_leaves=None, flags=0, nodes=None):
        """(n, 32) uint8 leaf digests -> (inner nodes (P - 1, 32) in heap order, root (32,))"""
        if not isinstance(leaves, (int, np.integer)):
            leaves = np.ascontiguousarray(leaves, dtype=np.uint8)
            n_leaves = leaves.shape[0]
        P = 1 << max(1, (n_leaves - 1).bit_length())
        if nodes is None:
            nodes = np.zeros((P - 1, 32), dtype=np.uint8)
        root = np.zeros(32, dtype=np.uint8)
        self._ck(self.lib.pcgpu_merkle_tree(self.ctx, _ptr(leaves), n_leaves, flags, _ptr(nodes), _ptr(root)))
        return nodes, root

    def lincode_commit(self, curve, mat, log_ext_cols, n_rows=None, n_cols=None, hash=0, flags=0, want=("ext", "leaves", "nodes"),
                       out_ext=None, out_leaves=None, out_nodes=None):
        """row encoding + column hashes + Merkle tree in one device-resident call -> dict(root, ext?, leaves?, nodes?)"""
        mat = _u64(mat)
        if n_rows is None:
            n_rows, n_cols = mat.shape[0], mat.shape[1]
        N = 1 << log_ext_cols
        if not (flags & DEVICE_PTRS):
            out_ext = np.zeros((n_rows, N, 4), dtype=np.uint64) if "ext" in want else None
            out_leaves = np.zeros((N, 32), dtype=np.uint8) if "leaves" in want else None
            out_nodes = np.zeros((N - 1, 32), dtype=np.uint8) if "nodes" in want else None
        root = np.zeros(32, dtype=np.uint8)
        self._ck(self.lib.pcgpu_lincode_commit(self.ctx, curve, _ptr(mat), n_rows, n_cols, log_ext_cols, hash, flags, _ptr(out_ext),
                                               _ptr(out_leaves), _ptr(out_nodes), _ptr(root)))
        return dict(root=root, ext=out_ext, leaves=out_leaves, nodes=out_nodes)

    # ---- multi-GPU over NVLink peer memory ----
    def peer_window_bytes(self):
        return int(self.lib.pcgpu_peer_window_bytes())

    def peer_alloc(self, nbytes):
        """zero-filled device buffer other processes can map -> (device pointer, 64-byte IPC handle)"""
        p, h = _vp(), np.zeros(64, dtype=np.uint8)
        self._ck(self.lib.pcgpu_peer_alloc(self.ctx, nbytes, ctypes.byref(p), _ptr(h)))
        return int(p.value), h

    def peer_open(self, handle):
        p, h = _vp(), np.ascontiguousarray(handle, dtype=np.uint8)
        self._ck(self.lib.pcgpu_peer_open(self.ctx, _ptr(h), ctypes.byref(p)))
        return int(p.value)

    def peer_close(self, ptr):
        self._ck(self.lib.pcgpu_peer_close(self.ctx, _vp(ptr)))

    def peer_free(self, ptr):
        self._ck(self.lib.pcgpu_peer_free(self.ctx, _vp(ptr)))

    def peer_signal(self, win, rank, channel, epoch):
        arr = (_vp * len(win))(*[ctypes.c_void_p(int(p)) for p in win])
        self._ck(self.lib.pcgpu_peer_signal(self.ctx, arr, rank, len(win), channel, epoch))

    def peer_wait(self, local_win, world, channel, epoch):
        self._ck(self.lib.pcgpu_peer_wait(self.ctx, _vp(int(local_win)), world, channel, epoch))

    def msm_peer(self, srs, scalars, win, rank, epoch, n=None, base_offset=0, flags=0):
        """this rank's slice of an index-sharded MSM; the point-sum over all ranks is fused into the call -> (xy, is_identity)"""
        scalars = _u64(scalars)
        if n is None:
            n = scalars.size // 4
        arr = (_vp * len(win))(*[ctypes.c_void_p(int(p)) for p in win])
        out = np.zeros(2 * fq_limbs(srs.curve), dtype=np.uint64)
        inf = np.zeros(1, dtype=np.uint8)
        self._ck(self.lib.pcgpu_msm_peer(self.ctx, srs.handle, base_offset, _ptr(scalars), n, flags, arr, rank, len(win), epoch,
                                         _ptr(out), _ptr(inf)))
        return out, int(inf[0])

    # ---- IPA halving loop (device-resident state) ----
    def ipa_begin(self, curve, comm_key_xy, coeffs, point, n=None, flags=0, n_coeffs=None):
        """comm_key_xy / coeffs: host arrays, or device pointers (ints) with DEVICE_PTRS -- a committer key that stays resident in
        a device buffer across openings, like a registered SRS -- in which case n and n_coeffs are required."""
        comm_key_xy, coeffs, point = _u64(comm_key_xy), _u64(coeffs), _u64(point)
        if n is None:
            n = comm_key_xy.size // (2 * fq_limbs(curve))
        if n_coeffs is None:
            n_coeffs = coeffs.size // 4
        h = _vp()
        self._ck(self.lib.pcgpu_ipa_begin(self.ctx, curve, _ptr(comm_key_xy), n, _ptr(coeffs), n_coeffs, _ptr(point), flags,
                                          ctypes.byref(h)))
        return IpaState(self, h, curve)

    def ipa_round_lr(self, curve, state, h_prime_xy, with_inf=False):
        h_prime_xy = _u64(h_prime_xy)
        nq = fq_limbs(curve)
        l, r = np.zeros(2 * nq, dtype=np.uint64), np.zeros(2 * nq, dtype=np.uint64)
        li, ri = np.zeros(1, dtype=np.uint8), np.zeros(1, dtype=np.uint8)
        self._ck(self.lib.pcgpu_ipa_round_lr(self.ctx, state.handle, _ptr(h_prime_xy), _ptr(l), _ptr(li), _ptr(r), _ptr(ri)))
        return (l, int(li[0]), r, int(ri[0])) if with_inf else (l, r)

    def ipa_round_fold(self, state, challenge, challenge_inv):
        self._ck(self.lib.pcgpu_ipa_round_fold(self.ctx, state.handle, _ptr(_u64(challenge)), _ptr(_u64(challenge_inv))))

    def ipa_len(self, state):
        return int(self.lib.pcgpu_ipa_len(state.handle)) if state.handle is not None else 0

    def ipa_check_final_key(self, comm_key_srs, challenges):
        """InnerProductArgPC::check's linear-time step: cm_commit(comm_key, check_poly.compute_coeffs())."""
        challenges = _u64(challenges)
        log_d = challenges.size // 4
        out = np.zeros(2 * fq_limbs(comm_key_srs.curve), dtype=np.uint64)
        inf = np.zeros(1, dtype=np.uint8)
        self._ck(self.lib.pcgpu_ipa_check_final_key(self.ctx, comm_key_srs.handle, _ptr(challenges), log_d, _ptr(out), _ptr(inf)))
        return out, int(inf[0])

    def ipa_finish(self, curve, state):
        """final_comm_key and c; releases the device state"""
        key, c = np.zeros(2 * fq_limbs(curve), dtype=np.uint64), np.zeros(4, dtype=np.uint64)
        h, state.handle = state.handle, None            # pcgpu_ipa_finish frees the state whatever it returns
        self._ck(self.lib.pcgpu_ipa_finish(self.ctx, h, _ptr(key), _ptr(c)))
        return key, c

    # ---- KZG10 ----
    def kzg_commit(self, powers_of_g, coeffs, n=None, powers_of_gamma_g=None, blind=None, flags=0):
        coeffs, blind = _u64(coeffs), _u64(blind)
        if n is None:
            n = coeffs.size // 4
        nb = 0 if blind is None else blind.size // 4
        out = np.zeros(2 * fq_limbs(powers_of_g.curve), dtype=np.uint64)
        inf = np.zeros(1, dtype=np.uint8)
        self._ck(self.lib.pcgpu_kzg_commit(self.ctx, powers_of_g.handle, _ptr(coeffs), n,
                                           None if powers_of_gamma_g is None else powers_of_gamma_g.handle,
                                           _ptr(blind), nb, flags, _ptr(out), _ptr(inf)))
        return out, int(inf[0])

    def kzg_commit_batch(self, powers_of_g, polys, flags=0):
        """MarlinKZG10::commit's loop over polynomials (marlin_pc/mod.rs:192-241), non-hiding: list of coefficient arrays
        (or (device_ptr, n) tuples with DEVICE_PTRS) -> ((count, 2*limbs) uint64, (count,) uint8)."""
        count = len(polys)
        ptrs, lens, keep = (ctypes.c_void_p * count)(), (_sz * count)(), []
        for i, p in enumerate(polys):
            if isinstance(p, tuple):
                ptrs[i], lens[i] = int(p[0]), int(p[1])
            else:
                a = _u64(p); keep.append(a)
                ptrs[i], lens[i] = a.ctypes.data, a.size // 4
        out = np.zeros((count, 2 * fq_limbs(powers_of_g.curve)), dtype=np.uint64)
        inf = np.zeros(count, dtype=np.uint8)
        self._ck(self.lib.pcgpu_kzg_commit_batch(self.ctx, powers_of_g.handle, ptrs, lens, count, flags, _ptr(out), _ptr(inf)))
        return out, inf

    def kzg_commit_open(self, powers_of_g, coeffs, z, n=None, flags=0):
        """KZG10::commit + KZG10::open of one polynomial in one call (coefficients uploaded once, the two MSMs overlapped)
        -> ((comm_xy, comm_is_identity), (w_xy, w_is_identity))"""
        coeffs, z = _u64(coeffs), _u64(z)
        if n is None:
            n = coeffs.size // 4
        nq = 2 * fq_limbs(powers_of_g.curve)
        c, w = np.zeros(nq, dtype=np.uint64), np.zeros(nq, dtype=np.uint64)
        ci, wi = np.zeros(1, dtype=np.uint8), np.zeros(1, dtype=np.uint8)
        self._ck(self.lib.pcgpu_kzg_commit_open(self.ctx, powers_of_g.handle, _ptr(coeffs), n, _ptr(z), flags, _ptr(c), _ptr(ci),
                                                _ptr(w), _ptr(wi)))
        return (c, int(ci[0])), (w, int(wi[0]))

    def kzg_commit_open_batch(self, powers_of_g, polys, z, flags=0):
        """commit + open of `count` polynomials at the same point (list of arrays, or (device_ptr, n) tuples with
        DEVICE_PTRS) -> (comm (count, 2*limbs), comm_inf (count,), w (count, 2*limbs), w_inf (count,))"""
        count = len(polys)
        ptrs, lens, keep = (ctypes.c_void_p * count)(), (_sz * count)(), []
        for i, p in enumerate(polys):
            if isinstance(p, tuple):
                ptrs[i], lens[i] = int(p[0]), int(p[1])
            else:
                a = _u64(p); keep.append(a)
                ptrs[i], lens[i] = a.ctypes.data, a.size // 4
        nq = 2 * fq_limbs(powers_of_g.curve)
        c, w = np.zeros((count, nq), dtype=np.uint64), np.zeros((count, nq), dtype=np.uint64)
        ci, wi = np.zeros(count, dtype=np.uint8), np.zeros(count, dtype=np.uint8)
        self._ck(self.lib.pcgpu_kzg_commit_open_batch(self.ctx, powers_of_g.handle, ptrs, lens, count, _ptr(_u64(z)), flags, _ptr(c),
                                                      _ptr(ci), _ptr(w), _ptr(wi)))
        return c, ci, w, wi

    def kzg_open(self, powers_of_g, coeffs, z, n=None, powers_of_gamma_g=None, blind=None, flags=0):
        coeffs, blind, z = _u64(coeffs), _u64(blind), _u64(z)
        if n is None:
            n = coeffs.size // 4
        nb = 0 if blind is None else blind.size // 4
        out = np.zeros(2 * fq_limbs(powers_of_g.curve), dtype=np.uint64)
        inf = np.zeros(1, dtype=np.uint8)
        rv = np.zeros(4, dtype=np.uint64)
        self._ck(self.lib.pcgpu_kzg_open(self.ctx, powers_of_g.handle, _ptr(coeffs), n, _ptr(z),
                                         None if powers_of_gamma_g is None else powers_of_gamma_g.handle,
                                         _ptr(blind), nb, flags, _ptr(out), _ptr(inf), _ptr(rv)))
        return out, int(inf[0]), (rv if nb else None)
