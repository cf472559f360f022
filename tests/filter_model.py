"""f64 models of the reference's f32 filters, written from the crate's source (src/svf.rs, src/biquad.rs, src/biquad_bank.rs,
src/moog.rs, src/filter.rs, src/rez.rs), each with an error bound per output sample that an f32 implementation of the same formulas must
stay within. numpy only.

Coefficients are evaluated as the crate writes them for F = f32: the f32 constants (F::from_f64(PI) is the f32 nearest pi), the order of
operations, and f32 inputs. They are evaluated in a tracked arithmetic `T`: an f64 value plus a first-order bound on how far the f32
evaluation of the same expression can be from it (Wilkinson style). + - * / and sqrt add half an ulp of their result (U = 2^-24 relative)
and 2^-149 absolute, since subnormals are kept; tanf, sinf, cosf and expf add one ulp of their result, tanhf two, and each passes on the
rounding of its argument through its own slope (the exact change over the argument's interval for the monotone ones).

The recurrences run in f64 from the coefficients' f64 values. The bound of output n sums, over every earlier step k, the local error of
step k (its rounding and its coefficients' error times the step's slope in each coefficient, from the same tracked arithmetic with the
state taken as exact) carried to output n through the exact Jacobians of the f64 trajectory:

    bound[n] = delta_y[n] + sum_k sum_j |C_n Phi(n, k+1) e_j| delta_x[k][j]

Each local error is propagated as its own column and absolute values are summed only at the output; an elementwise |A| recursion would
diverge for a resonant filter, whose |A| has spectral radius above 1. Moog, Rez and tanh are linearised around the trajectory. Columns
below 2^-60 of the running bound are dropped. A final factor 1 + 2^-10 covers the second-order terms.

`mutate=` builds a model with one deliberate mistake, as a negative control for the tests:
  "swap_a"      a1 and a2 swapped (SVF and biquad coefficients)
  "m1_sign"     m1 with the wrong sign (SVF modes whose m1 is not zero)
  "cutoff_only" coefficients recomputed on a cutoff change only, so a change of q or gain alone is ignored
  "late"        new coefficients applied one sample late
  "stale_rate"  set_sample_rate keeps the old rate's coefficients
  "no_ps"       Moog without its px / ps terms
  "rez_fb"      Rez's fb without the / (1 - f) term
"""
import math

import numpy as np

F32 = np.float32
U = 2.0 ** -24
FLOOR = 2.0 ** -149
SLACK = 1.0 + 2.0 ** -10
DEFAULT_SR = 44100.0
PI = float(F32(math.pi))           # F::PI, F::from_f64(f64::PI) for F = f32
TAU = float(F32(2.0 * math.pi))    # F::TAU
SQRT_2 = float(F32(math.sqrt(2.0)))
MODES = ("lowpass", "highpass", "bandpass", "notch", "peak", "allpass", "bell", "lowshelf", "highshelf")


def f32(x):
    return float(F32(x))


def ulp(v):
    """One f32 ulp of |v| (2^-149 at and below the subnormal range)."""
    v = np.abs(np.asarray(v, np.float64))
    with np.errstate(over="ignore", invalid="ignore"):
        _, e = np.frexp(v)
        return np.where(np.isfinite(v), np.ldexp(1.0, np.maximum(e.astype(np.int64) - 24, -149)), np.inf)


class T:
    """A value computed in f32, as (v, e): v its f64 value, e a bound on |f32 result - v|. Works elementwise on numpy arrays."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v, self.e = v, e

    @staticmethod
    def of(x):
        return x if isinstance(x, T) else T(x, 0.0)

    @staticmethod
    def _r(v, e):   # round the result: half an ulp of the computed value, and the subnormal floor
        with np.errstate(over="ignore", invalid="ignore"):
            return T(v, e + U * (np.abs(v) + e) + FLOOR)

    def __add__(self, o):
        o = T.of(o)
        return T._r(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = T.of(o)
        return T._r(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return T.of(o) - self

    def __neg__(self):
        return T(-self.v, self.e)

    def __mul__(self, o):
        o = T.of(o)
        with np.errstate(over="ignore", invalid="ignore"):
            return T._r(self.v * o.v, np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = T.of(o)
        with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
            v = self.v / o.v
            den = np.abs(o.v) - o.e
            e = np.where(den > 0, (self.e + np.abs(v) * o.e) / np.where(den > 0, den, 1.0), np.inf)
        return T._r(v, e)

    def __rtruediv__(self, o):
        return T.of(o) / self


def _monotone(fn, a, ulps):
    """fn (monotone on the argument's interval) of a T: the change over [v - e, v + e], plus `ulps` ulps of the result."""
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        v = fn(a.v)
        e = np.maximum(np.abs(fn(a.v + a.e) - v), np.abs(fn(a.v - a.e) - v))
        e = np.where(np.isnan(e) & np.isfinite(v), np.inf, e)
        return T(v, e + ulps * ulp(np.abs(v) + e) + FLOOR)


def tan(a):
    with np.errstate(invalid="ignore"):   # an interval that reaches a pole of tan has no bound
        k = np.floor((np.asarray(a.v) - a.e) / math.pi + 0.5) != np.floor((np.asarray(a.v) + a.e) / math.pi + 0.5)
    r = _monotone(np.tan, a, 1.0)
    return T(r.v, np.where(k, np.inf, r.e))


def exp(a):
    return _monotone(np.exp, a, 1.0)


def sqrt(a):
    r = _monotone(np.sqrt, a, 0.5)
    return T(r.v, np.where(np.asarray(a.v) - a.e < 0, np.inf, r.e))


def tanh(a):
    return _monotone(np.tanh, a, 2.0)


def sin(a):   # |sin'| <= 1
    with np.errstate(invalid="ignore"):
        v = np.sin(a.v)
        return T(v, np.minimum(a.e, 2.0) + ulp(np.abs(v) + a.e) + FLOOR)


def cos(a):
    with np.errstate(invalid="ignore"):
        v = np.cos(a.v)
        return T(v, np.minimum(a.e, 2.0) + ulp(np.abs(v) + a.e) + FLOOR)


# ---------------------------------------------------------------- coefficients
def svf_coefs(mode, sr, cutoff, q, gain, mutate=None):
    """src/svf.rs:26-221 (SvfCoefs::lowpass ... highshelf) for F = f32. Returns (a1, a2, a3, m0, m1, m2) as T."""
    one = 1.0
    sr, cutoff, q, gain = T.of(sr), T.of(cutoff), T.of(q), T.of(gain)
    if mode in ("bell", "lowshelf", "highshelf"):
        a = sqrt(gain)
    g = tan(PI * cutoff / sr)
    if mode == "lowshelf":
        g = g / sqrt(a)
    elif mode == "highshelf":
        g = g * sqrt(a)
    k = one / (q * a) if mode == "bell" else one / q
    a1 = one / (one + g * (g + k))
    a2 = g * a1
    a3 = g * a2
    z, o = T(0.0 * cutoff.v), T(0.0 * cutoff.v + 1.0)
    m0, m1, m2 = {
        "lowpass": lambda: (z, z, o),
        "highpass": lambda: (o, -k, -o),
        "bandpass": lambda: (z, o, z),
        "notch": lambda: (o, -k, z),
        "peak": lambda: (o, -k, T(0.0 * cutoff.v - 2.0)),
        "allpass": lambda: (o, -2.0 * k, z),
        "bell": lambda: (o, k * (a * a - one), z),
        "lowshelf": lambda: (o, k * (a - one), a * a - one),
        "highshelf": lambda: (a * a, k * (one - a) * a, one - a * a),
    }[mode]()
    if mutate == "swap_a":
        a1, a2 = a2, a1
    if mutate == "m1_sign":
        m1 = -m1
    return a1, a2, a3, m0, m1, m2


def butter_lowpass(sr, cutoff):
    """src/biquad.rs:27-38, BiquadCoefs::butter_lowpass. Returns (a1, a2, b0, b1, b2)."""
    f = tan(T.of(cutoff) * PI / sr)
    a0r = 1.0 / (1.0 + SQRT_2 * f + f * f)
    a1 = (2.0 * f * f - 2.0) * a0r
    a2 = (1.0 - SQRT_2 * f + f * f) * a0r
    b0 = f * f * a0r
    return a1, a2, b0, 2.0 * b0, b0


def resonator(sr, center, q):
    """src/biquad.rs:40-50, BiquadCoefs::resonator."""
    center = T.of(center)
    r = exp(-PI * center / (T.of(q) * sr))
    a1 = -2.0 * r * cos(TAU * center / sr)
    a2 = r * r
    b0 = sqrt(1.0 - r * r) * 0.5
    return a1, a2, b0, T(0.0 * center.v), -b0


def moog_coefs(sr, cutoff, q):
    """src/moog.rs:48-57, Moog::set_cutoff_q. Returns (p, k, rez)."""
    c = 2.0 * T.of(cutoff) / sr
    p = c * (f32(1.8) - f32(0.8) * c)
    k = 2.0 * sin(c * PI * 0.5) - 1.0
    t1 = (1.0 - p) * f32(1.386249)
    t2 = 12.0 + t1 * t1
    rez = T.of(q) * (t2 + 6.0 * t1) / (t2 - 6.0 * t1)
    return p, k, rez


def rez_coefs(sr, cutoff, q, mutate=None):
    """src/rez.rs:41-46, Rez::set_cutoff_q. Returns (f, fb)."""
    f = 2.0 * sin(PI * T.of(cutoff) / sr)
    q = T.of(q)
    fb = q + q if mutate == "rez_fb" else q + q / (1.0 - f)
    return f, fb


def onepole_coef(kind, sr, p):
    """src/filter.rs: Lowpole / Highpole exp(-TAU cutoff / sr) (:43-46, :376-379), Allpole (1 - d) / (1 + d) (:294-296), DCBlock
    1 - TAU / sr * cutoff (:123-126)."""
    p = T.of(p)
    if kind in ("lowpole", "highpole"):
        return (exp(-TAU * p / sr),)
    if kind == "allpole":
        return ((1.0 - p) / (1.0 + p),)
    return (1.0 - TAU / T.of(sr) * p,)


# ---------------------------------------------------------------- one step of each node, generic over float / Dual / T
# state layouts: svf (ic1, ic2); biquad (x1, x2, y1, y2); lowpole (y1,); highpole / allpole / dcblock (x1, y1);
# moog (s0, s1, s2, s3, px, ps0, ps1, ps2); rez (buf0, buf1). Each returns (new state, output).
def step_svf(s, x, k):   # src/svf.rs:829-838 (Svf::tick), :995-1006 (FixedSvf::tick)
    ic1, ic2 = s
    a1, a2, a3, m0, m1, m2 = k
    v3 = x - ic2
    v1 = a1 * ic1 + a2 * v3
    v2 = ic2 + a2 * ic1 + a3 * v3
    return (2.0 * v1 - ic1, 2.0 * v2 - ic2), m0 * x + m1 * v1 + m2 * v2


def step_biquad(s, x, k):   # src/biquad.rs:184-194
    x1, x2, y1, y2 = s
    a1, a2, b0, b1, b2 = k
    y0 = b0 * x + b1 * x1 + b2 * x2 - a1 * y1 - a2 * y2
    return (x, x1, y0, y1), y0


def step_onepole(kind):
    def lowpole(s, x, k):   # src/filter.rs:64-75
        (c,) = k
        y = (1.0 - c) * x + c * s[0]
        return (y,), y

    def highpole(s, x, k):   # :398-409
        (c,) = k
        y = c * (s[1] + x - s[0])
        return (x, y), y

    def allpole(s, x, k):   # :314-323
        (eta,) = k
        y = eta * (x - s[1]) + s[0]
        return (x, y), y

    def dcblock(s, x, k):   # :145-151
        (c,) = k
        y = x - s[0] + c * s[1]
        return (x, y), y
    return {"lowpole": lowpole, "highpole": highpole, "allpole": allpole, "dcblock": dcblock}[kind]


def step_moog(mutate):
    def step(s, x, k):   # src/moog.rs:87-98
        s0, s1, s2, s3, px, ps0, ps1, ps2 = s
        p, kk, rez = k
        if mutate == "no_ps":
            px = ps0 = ps1 = ps2 = 0.0 * x
        xx = -rez * s3 + x
        s0 = (xx + px) * p - kk * s0
        s1 = (s0 + ps0) * p - kk * s1
        s2 = (s1 + ps1) * p - kk * s2
        s3 = _tanh((s2 + ps2) * p - kk * s3)
        return (s0, s1, s2, s3, xx, s0, s1, s2), s3
    return step


def step_rez(bandpass):
    def step(s, x, k):   # src/rez.rs:65-79
        buf0, buf1 = s
        f, fb = k
        hp = x - buf0
        bp = buf0 - buf1
        buf0 = buf0 + f * (hp + fb * _tanh(bp))
        buf1 = buf1 + f * (buf0 - buf1)
        return (buf0, buf1), buf1 - bandpass * buf0
    return step


class Dual:
    """A value and its gradient over the state (forward mode): gives the exact Jacobians of a step at the f64 trajectory."""
    __slots__ = ("v", "g")

    def __init__(self, v, g):
        self.v, self.g = v, g

    @staticmethod
    def of(x, d):
        return x if isinstance(x, Dual) else Dual(float(x), np.zeros(d))

    def __add__(self, o):
        o = Dual.of(o, self.g.size)
        return Dual(self.v + o.v, self.g + o.g)

    __radd__ = __add__

    def __sub__(self, o):
        o = Dual.of(o, self.g.size)
        return Dual(self.v - o.v, self.g - o.g)

    def __rsub__(self, o):
        return Dual.of(o, self.g.size) - self

    def __neg__(self):
        return Dual(-self.v, -self.g)

    def __mul__(self, o):
        o = Dual.of(o, self.g.size)
        return Dual(self.v * o.v, self.g * o.v + o.g * self.v)

    __rmul__ = __mul__


def _tanh(a):
    if isinstance(a, T):
        return tanh(a)
    if isinstance(a, Dual):
        t = math.tanh(a.v)
        return Dual(t, a.g * (1.0 - t * t))
    return np.tanh(a)


# ---------------------------------------------------------------- the units
FAMILIES = MODES + ("morph", "butterpass", "resonator", "biquad", "lowpole", "highpole", "allpole", "dcblock", "moog", "lowrez", "bandrez")
DIM = dict({m: 2 for m in MODES}, morph=2, butterpass=4, resonator=4, biquad=4, lowpole=1, highpole=2, allpole=2, dcblock=2, moog=8,
           lowrez=2, bandrez=2)
NCTL = dict({m: (3 if i >= 6 else 2) for i, m in enumerate(MODES)}, morph=3, butterpass=1, resonator=2, biquad=0, lowpole=1,
            highpole=1, allpole=1, dcblock=1, moog=2, lowrez=2, bandrez=2)


class Unit:
    """One filter node as the reference runs it (tick by tick): `fam` one of FAMILIES; `params` its constructor values (cutoff /
    center, q, gain for the SVFs; morph's third is its morph input, not a parameter; biquad: (a1, a2, b0, b1, b2)); `fixed` the *_hz
    form, whose coefficients change only with the rate. `run(x, ctl)` continues from the current state and returns (f64 output, bound)."""

    def __init__(self, fam, params=(440.0, 1.0, 1.0), fixed=False, mutate=None):
        assert fam in FAMILIES, fam
        self.fam, self.fixed, self.mutate = fam, fixed or fam == "biquad", mutate
        self.sr = DEFAULT_SR
        self.params = tuple(f32(p) for p in params)
        if fam == "allpole" and len(params) == 3:
            self.params = (1.0,)
        self.d = DIM[fam]
        self.state = np.zeros(self.d)
        self.E = np.zeros((self.d, 0))
        self.k = self._coefs(self.params)

    # coefficients from (cutoff, q, gain) at the current rate, as T tuples
    def _coefs(self, p, sr=None):
        sr = f32(self.sr if sr is None else sr)
        fam, mut = self.fam, self.mutate
        p = tuple(np.asarray(v, np.float64) for v in p)
        if fam in MODES:
            return svf_coefs(fam, sr, p[0], p[1], p[2] if len(p) > 2 else 1.0, mut)
        if fam == "morph":
            return svf_coefs("peak", sr, p[0], p[1], 1.0, mut)
        if fam == "butterpass":
            k = butter_lowpass(sr, p[0])
        elif fam == "resonator":
            k = resonator(sr, p[0], p[1])
        elif fam == "biquad":
            k = tuple(T(v) for v in p)
        elif fam == "moog":
            return moog_coefs(sr, p[0], p[1])
        elif fam in ("lowrez", "bandrez"):
            return rez_coefs(sr, p[0], p[1], mut)
        else:
            return onepole_coef(fam, sr, p[0])
        if mut == "swap_a":
            k = (k[1], k[0]) + tuple(k[2:])
        return k

    def set_sample_rate(self, sr):
        """src/svf.rs:823-826, src/biquad.rs:263-266 / :349-351, src/filter.rs:58-61 / :392-395, src/rez.rs:59-62, src/moog.rs:76-79:
        the coefficients are recomputed from the stored parameters (Allpole's do not depend on the rate)."""
        self.sr = sr
        if self.mutate != "stale_rate" and self.fam != "biquad":
            self.k = self._coefs(self.params)

    def reset(self):
        self.state = np.zeros(self.d)
        self.E = np.zeros((self.d, 0))

    def _step(self):
        fam = self.fam
        if fam in MODES or fam == "morph":
            return step_svf
        if fam in ("butterpass", "resonator", "biquad"):
            return step_biquad
        if fam == "moog":
            return step_moog(self.mutate)
        if fam in ("lowrez", "bandrez"):
            return step_rez(0.0 if fam == "lowrez" else 1.0)
        return step_onepole(fam)

    def _schedule(self, ctl, n):
        """Coefficients in effect at every sample: (index into the recompute list per sample, list of parameter tuples)."""
        fam, mut = self.fam, self.mutate
        nc = NCTL[fam] if not self.fixed else 0
        if fam == "morph":
            nc = 2
        sets, idx = [self.params], np.zeros(n, np.int64)
        if nc == 0:
            return idx, sets
        c = [np.asarray(ctl[j], F32) for j in range(nc)]
        cur = list(self.params)
        for i in range(n):
            v = [float(c[j][i]) for j in range(nc)]
            if fam == "moog" or fam == "allpole":   # src/moog.rs:83-85 and src/filter.rs:315-317: every sample
                ch = True
            elif mut == "cutoff_only":
                ch = v[0] != cur[0]
            else:
                ch = any(v[j] != cur[j] for j in range(nc))
            if ch:
                cur = v + list(cur[nc:])
                sets.append(tuple(cur))
            idx[i] = len(sets) - 1
        self.params = tuple(cur)
        return idx, sets

    def run(self, x, ctl=()):
        x = np.asarray(x, F32).astype(np.float64)
        n = x.size
        idx, sets = self._schedule(ctl, n)
        vals = [np.array([float(np.asarray(k.v))]) for k in self.k]
        errs = [np.array([float(np.asarray(k.e))]) for k in self.k]
        if len(sets) > 1:
            k1 = self._coefs([np.array([st[j] for st in sets[1:]]) for j in range(len(sets[1]))])
            for j, k in enumerate(k1):
                vals[j] = np.concatenate([vals[j], np.broadcast_to(k.v, (len(sets) - 1,))])
                errs[j] = np.concatenate([errs[j], np.broadcast_to(k.e, (len(sets) - 1,))])
        use = np.concatenate([[0], idx[:-1]]) if self.mutate == "late" else idx   # "late": sample i on the coefficients of i - 1
        ks = [(v[use], e[use]) for v, e in zip(vals, errs)]
        if n:
            self.k = tuple(T(v[idx[-1]], e[idx[-1]]) for v, e in zip(vals, errs))
        step, d = self._step(), self.d
        # the f64 trajectory, and the Jacobians of state and output at every step
        S = np.empty((n, d))
        A = np.empty((n, d, d))
        Cm = np.empty((n, d))
        y = np.empty(n)
        s = self.state.copy()
        eye = np.eye(d)
        for i in range(n):
            S[i] = s
            kv = tuple(kk[0][i] for kk in ks)
            if np.all(np.isfinite(s)) and all(math.isfinite(v) for v in kv):
                ns, out = step(tuple(Dual(s[j], eye[j]) for j in range(d)), x[i], kv)
                s = np.array([Dual.of(v, d).v for v in ns])
                A[i] = np.array([Dual.of(v, d).g for v in ns])
                out = Dual.of(out, d)
                y[i], Cm[i] = out.v, out.g
            else:
                s = np.full(d, np.nan)
                A[i], Cm[i], y[i] = np.nan, np.nan, np.nan
        self.state = s
        # local errors: the step in the tracked arithmetic with the state exact and the coefficients as computed
        with np.errstate(over="ignore", invalid="ignore"):
            ns, out = step(tuple(T(S[:, j]) for j in range(d)), T(x), tuple(T(v, e) for v, e in ks))
        dx = np.stack([np.broadcast_to(T.of(v).e, (n,)) for v in ns], axis=1) if n else np.zeros((0, d))
        dy = np.broadcast_to(T.of(out).e, (n,)).copy()
        if self.fam == "morph":   # src/svf.rs:1077-1081: (filter + morph * x) * 0.5
            m = np.asarray(ctl[2], F32).astype(np.float64)
            with np.errstate(over="ignore", invalid="ignore"):
                yt = T(y, dy) + T(m) * T(x)
                dy = 0.5 * yt.e
                y = 0.5 * (y + m * x)
            Cm = 0.5 * Cm
        bound = np.empty(n)
        E = np.zeros((d, self.E.shape[1] + d * n))
        E[:, :self.E.shape[1]] = self.E
        m = self.E.shape[1]
        with np.errstate(over="ignore", invalid="ignore"):
            for i in range(n):
                b = dy[i] + float(np.abs(Cm[i] @ E[:, :m]).sum())
                bound[i] = b
                E[:, :m] = A[i] @ E[:, :m]
                E[:, m:m + d] = np.diag(dx[i])
                m += d
                if i % 256 == 255 and np.isfinite(b):   # drop the columns that no longer reach 2^-60 of the bound
                    keep = np.abs(E[:, :m]).max(axis=0) >= 2.0 ** -60 * max(b, FLOOR)
                    kept = int(keep.sum())
                    E[:, :kept] = E[:, :m][:, keep]
                    m = kept
        self.E = E[:, :m].copy()
        return y, bound * SLACK


def run(fam, x, ctl=(), sr=48000.0, params=None, fixed=False, mutate=None):
    """A unit constructed with `params` (default: the prelude's constructor values), set to `sr`, run over x and the control rows."""
    if params is None:
        params = {"morph": (440.0, 1.0, 1.0), "moog": (1000.0, 0.1, 1.0), "allpole": (1.0,)}.get(fam, (440.0, 1.0, 1.0))
    u = Unit(fam, params, fixed=fixed, mutate=mutate)
    u.set_sample_rate(sr)
    return u.run(x, ctl)
