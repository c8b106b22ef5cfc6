"""TEST INFRASTRUCTURE -- an independent, definition-level optimal-ate pairing in Python big integers.

Not product code, and deliberately not the device's tower: Fq12 is one flat extension Fq[w]/(w^12 - c6 w^6 + c0),
  BLS12-381  w^12 - 2 w^6 + 2    (u = w^6 - 1, so w^6 = 1 + u = xi)
  BN254      w^12 - 18 w^6 + 82  (u = w^6 - 9, so w^6 = 9 + u = xi)
with inverses by the extended Euclidean algorithm over Fq[w].  A G2 point Q on the sextic twist is untwisted into E(Fq12),
  BN254 (D-type twist)      psi(x, y) = (x w^2, y w^3)
  BLS12-381 (M-type twist)  psi(x, y) = (x / w^2, y / w^3)
and the Miller loop runs in affine coordinates with chord and tangent lines evaluated at P; vertical lines are dropped, since
the final exponentiation maps them to 1.  The loop parameters are the curves' own:
  BLS12-381  |x| = 0xd201000000010000, then f -> f^(p^6) because x < 0
  BN254      6u + 2, then the lines through pi(Q) and -pi^2(Q) (pi: the p-power Frobenius)
The final exponentiation is pow(f, (p^12 - 1) / r) on the flat element.

to_tower / from_tower convert between the flat form and the byte layout of the device's tower
Fq12 = Fq6[w]/(w^2 - v), Fq6 = Fq2[v]/(v^3 - xi): twelve Fq coefficients c0.c0.c0, c0.c0.c1, c0.c1.c0 ... c1.c2.c1.
"""
import numpy as np

from oracle import pyref

_SPEC = {"bls12_381": dict(k=1, c6=2, c0=2, loop=0xd201000000010000, neg=True),
         "bn254": dict(k=9, c6=18, c0=82, loop=6 * 4965661367192848881 + 2, neg=False)}


class Pairing:
    def __init__(self, name):
        s = _SPEC[name]
        self.name = name
        self.C = pyref.Curve(name)
        self.G2 = pyref.G2(name)
        self.p, self.r = self.C.p, self.C.r
        self.k, self.c6, self.c0 = s["k"], s["c6"], s["c0"]
        self.loop, self.neg = s["loop"], s["neg"]
        p = self.p
        self.ONE = (1,) + (0,) * 11
        self.W = (0, 1) + (0,) * 10
        # w^-1 = (c6 w^5 - w^11) / c0, from w (w^11 - c6 w^5) = -c0
        ic0 = pow(self.c0, -1, p)
        winv = [0] * 12
        winv[5], winv[11] = self.c6 * ic0 % p, (-ic0) % p
        self.WINV = tuple(winv)
        assert self.mul(self.W, self.WINV) == self.ONE

    # ---- Fq12 = Fq[w] / (w^12 - c6 w^6 + c0) ----
    def add(self, a, b):
        p = self.p
        return tuple((x + y) % p for x, y in zip(a, b))

    def sub(self, a, b):
        p = self.p
        return tuple((x - y) % p for x, y in zip(a, b))

    def scal(self, a, s):
        p = self.p
        return tuple(x * s % p for x in a)

    def _reduce(self, t):
        p = self.p
        for i in range(len(t) - 1, 11, -1):        # w^i = w^(i-12) (c6 w^6 - c0)
            c = t[i]
            if c:
                t[i - 6] += self.c6 * c
                t[i - 12] -= self.c0 * c
            t[i] = 0
        return tuple(x % p for x in t[:12])

    def mul(self, a, b):
        t = [0] * 23
        for i, x in enumerate(a):
            if x:
                for j, y in enumerate(b):
                    t[i + j] += x * y
        return self._reduce(t)

    def pow(self, a, e):
        acc = self.ONE
        for bit in bin(e)[2:] if e else "":
            acc = self.mul(acc, acc)
            if bit == "1":
                acc = self.mul(acc, a)
        return acc

    def inv(self, a):
        """a^-1 by the extended Euclidean algorithm over Fq[w]; 0 -> 0"""
        p = self.p
        if not any(a):
            return (0,) * 12

        def trim(f):
            while f and f[-1] == 0:
                f.pop()
            return f

        def pdivmod(f, g):
            f, q = list(f), [0] * max(len(f) - len(g) + 1, 1)
            ig = pow(g[-1], -1, p)
            while len(trim(f)) >= len(g):
                c, d = f[-1] * ig % p, len(f) - len(g)
                q[d] = c
                for i, y in enumerate(g):
                    f[i + d] = (f[i + d] - c * y) % p
            return q, f

        def pmul(f, g):
            t = [0] * (len(f) + len(g))
            for i, x in enumerate(f):
                for j, y in enumerate(g):
                    t[i + j] = (t[i + j] + x * y) % p
            return trim(t)

        def psub(f, g):
            n = max(len(f), len(g))
            return trim([((f[i] if i < len(f) else 0) - (g[i] if i < len(g) else 0)) % p for i in range(n)])

        m = [self.c0, 0, 0, 0, 0, 0, (-self.c6) % p, 0, 0, 0, 0, 0, 1]
        r0, r1, s0, s1 = m, trim(list(a)), [], [1]
        while r1:
            q, rem = pdivmod(r0, r1)
            r0, r1, s0, s1 = r1, trim(rem), s1, psub(s0, pmul(q, s1))
        assert len(r0) == 1, "not invertible"
        c = pow(r0[0], -1, p)
        out = [x * c % p for x in s0] + [0] * 12
        return tuple(out[:12])

    def conj(self, a):
        """a^(p^6): w -> -w (w^(p^6) = -w, the coefficients are in Fq)"""
        p = self.p
        return tuple(x if i % 2 == 0 else (-x) % p for i, x in enumerate(a))

    def frob(self, a):
        return self.pow(a, self.p)

    def fq(self, x):
        return (x % self.p,) + (0,) * 11

    def fq2(self, z):
        """c0 + c1 u with u = w^6 - k"""
        p = self.p
        return ((z[0] - self.k * z[1]) % p,) + (0,) * 5 + (z[1] % p,) + (0,) * 5

    # ---- the curve E(Fq12): y^2 = x^3 + b ----
    def untwist(self, Q):
        if Q is None:
            return None
        x, y = self.fq2(Q[0]), self.fq2(Q[1])
        if self.name == "bn254":
            w2 = self.mul(self.W, self.W)
            return self.mul(x, w2), self.mul(y, self.mul(w2, self.W))
        wi2 = self.mul(self.WINV, self.WINV)
        return self.mul(x, wi2), self.mul(y, self.mul(wi2, self.WINV))

    def on_curve(self, P):
        x, y = P
        return self.sub(self.mul(y, y), self.mul(self.mul(x, x), x)) == self.fq(self.C.b)

    def _step(self, T, R, xP, yP):
        """(T + R, the line through T and R (tangent when T = R) at (xP, yP), or None for a vertical line)"""
        x1, y1 = T
        x2, y2 = R
        if x1 == x2:
            if self.add(y1, y2) == (0,) * 12:
                return None, None
            lam = self.mul(self.scal(self.mul(x1, x1), 3), self.inv(self.scal(y1, 2)))
        else:
            lam = self.mul(self.sub(y2, y1), self.inv(self.sub(x2, x1)))
        x3 = self.sub(self.sub(self.mul(lam, lam), x1), x2)
        y3 = self.sub(self.mul(lam, self.sub(x1, x3)), y1)
        line = self.sub(self.sub(yP, y1), self.mul(lam, self.sub(xP, x1)))
        return (x3, y3), line

    def miller(self, P, Q):
        """the optimal-ate Miller value of one pair (1 when P or Q is the identity)"""
        if P is None or Q is None:
            return self.ONE
        xP, yP = self.fq(P[0]), self.fq(P[1])
        Qt = self.untwist(Q)
        f, T = self.ONE, Qt
        for bit in bin(self.loop)[3:]:
            T2, l = self._step(T, T, xP, yP)
            f = self.mul(f, f)
            if l is not None:
                f = self.mul(f, l)
            T = T2
            if bit == "1":
                T2, l = self._step(T, Qt, xP, yP)
                if l is not None:
                    f = self.mul(f, l)
                T = T2
        if self.neg:
            f = self.conj(f)
        if self.name == "bn254":
            Q1 = (self.frob(Qt[0]), self.frob(Qt[1]))
            Q2 = (self.frob(Q1[0]), self.sub((0,) * 12, self.frob(Q1[1])))
            for R in (Q1, Q2):
                T2, l = self._step(T, R, xP, yP)
                if l is not None:
                    f = self.mul(f, l)
                T = T2
        return f

    def final_exp(self, f):
        return self.pow(f, (self.p ** 12 - 1) // self.r)

    def multi_pairing(self, Ps, Qs):
        f = self.ONE
        for P, Q in zip(Ps, Qs):
            f = self.mul(f, self.miller(P, Q))
        return self.final_exp(f)

    def pairing(self, P, Q):
        return self.multi_pairing([P], [Q])

    # ---- the device's tower layout ----
    def to_tower(self, a):
        """flat -> 12 Fq ints in ark order: g0, g2, g4 (c0), g1, g3, g5 (c1), each g_i = (re, im) with a = sum g_i w^i"""
        p, out = self.p, []
        for i in (0, 2, 4, 1, 3, 5):
            im = a[i + 6]
            out += [(a[i] + self.k * im) % p, im]
        return out

    def from_tower(self, t):
        p, a = self.p, [0] * 12
        for slot, i in enumerate((0, 2, 4, 1, 3, 5)):
            re, im = t[2 * slot], t[2 * slot + 1]
            a[i], a[i + 6] = (re - self.k * im) % p, im % p
        return tuple(a)

    def to_limbs(self, elems):
        """flat elements -> (n, 12 nq) uint64, Montgomery tower coefficients"""
        C = self.C
        out = np.zeros((len(elems), 12 * C.nq), dtype=np.uint64)
        for n, a in enumerate(elems):
            for s, c in enumerate(self.to_tower(a)):
                v = c * C.Rq % C.p
                for j in range(C.nq):
                    out[n, s * C.nq + j] = (v >> (64 * j)) & 0xFFFFFFFFFFFFFFFF
        return out

    def from_limbs(self, arr):
        C = self.C
        arr = np.asarray(arr, dtype=np.uint64).reshape(-1, 12 * C.nq)
        return [self.from_tower([sum(int(row[s * C.nq + j]) << (64 * j) for j in range(C.nq)) * C.Rq_inv % C.p
                                 for s in range(12)]) for row in arr]

    def random(self, g):
        return tuple(int.from_bytes(g.bytes(8 * self.C.nq), "little") % self.p for _ in range(12))
