"""f64 models of the reference's delay-line nodes — TEST INFRASTRUCTURE (numpy only; imports neither the oracle nor the product).

Each model is written from the fundsp crate's source (src/delay.rs, src/feedback.rs, src/oversample.rs), not from the oracle or the
product, so that a misreading the two share shows up against it. Every model takes the node's input samples (f32) and returns its
output in f64 together with a per-sample error bound: what an f32 evaluation of the same arithmetic may differ from the f64 value,
derived from the operation count (DESIGN §4). `mutate` applies one deliberate error to a model; the tests use it as a negative
control (a mutated model must miss the bound by orders of magnitude).
"""
import json
import os

import numpy as np

U = 2.0 ** -24
F32 = np.float32
SIMD_N = 8   # src/lib.rs SIMD_N: Tap's ring has room for one SIMD group of writes ahead of the oldest tap


def next_pow2(n):
    return 1 << max(0, int(n) - 1).bit_length()


def round_half_away(x):
    """Rust's f64::round: ties away from zero (numpy's rint rounds ties to even)."""
    return float(np.sign(x) * np.floor(abs(x) + 0.5))


# ---------------------------------------------------------------- Delay (src/delay.rs, ID 13)
def delay_samples(t, sr):
    """Delay::set_sample_rate: time_in_samples = round(t * sr) (f64, half away from zero); the ring holds one sample more."""
    return int(round_half_away(t * sr))


def delay(x, t, sr, mutate=None):
    """y[n] = x[n - L], zeros before the start. Delay::tick writes at i, advances i, and reads the oldest slot of a ring of L + 1
    samples, which is the sample written L ticks ago. Exact: the bound is 0."""
    L = delay_samples(t, sr) + (1 if mutate == "offset" else 0)
    x = np.asarray(x, np.float64)
    y = np.zeros_like(x)
    y[L:] = x[: x.size - L] if L else x
    return y, np.zeros_like(x)


# ---------------------------------------------------------------- Tap / TapLinear (src/delay.rs, IDs 50 / 54)
def tap_params(min_delay, max_delay, sr, linear):
    """(sr, lo, hi, ring length) as Tap::set_sample_rate computes them, in f32: lo = max(min, 1.00001 / sr) and hi = max(max, 1.00001 / sr)
    for Tap (at least one sample of delay, so the newest tap y0 is never a sample not yet written); TapLinear clamps to [min, max] as
    given. Ring: next_power_of_two(ceil(max * sr) + 3 + SIMD_N) for Tap, next_power_of_two(ceil(max * sr) + 2) for TapLinear."""
    s = F32(sr)
    mn, mx = F32(min_delay), F32(max_delay)
    floor1 = F32(1.00001) / s
    lo, hi = (mn, mx) if linear else (max(mn, floor1), max(mx, floor1))
    extra = 2.0 if linear else 3.0 + SIMD_N
    ring = next_pow2(int(np.ceil(F32(mx * s)) + F32(extra)))
    return s, F32(lo), F32(hi), ring


def tap_positions(d, lo, hi, s):
    """D = clamp(d, lo, hi) * sr in f32. The clamp is Rust's `x.max(lo).min(hi)` (src/math.rs clamp): f32::max returns the other operand
    when one is NaN, so a NaN delay reads at lo; the block path's `fast_max` then `fast_min` gives the same. -inf and anything below lo
    read at lo, +inf and anything above hi at hi."""
    d = np.asarray(d, F32)
    c = np.where(np.isnan(d), lo, np.minimum(np.maximum(d, lo), hi)).astype(F32)
    with np.errstate(over="ignore"):
        return (c * s).astype(F32)


def tap(x, delays, min_delay, max_delay, sr, linear=False, mutate=None):
    """Tap<N> / TapLinear<N>: x the audio input, delays [N][n] the delay inputs in seconds. Returns (y, bound).

    The tap position D is f32 (floor(D) picks the samples, so it must round as the reference's does); the interpolation and the
    sum over taps are f64 over the input history, zeros before the start. With f = floor(D) and t = D - f (exact in f32):
      Tap:       spline(x[n-f+1], x[n-f], x[n-f-1], x[n-f-2], t)   (src/math.rs spline, Catmull-Rom between x[n-f] and x[n-f-1])
      TapLinear: lerp(x[n-f], x[n-f-1], t)
    This is the reference's `tick` path, and the product's and the oracle's in every context. The ring is not modelled: a ring too
    short for the taps, a wrong mask or a wrong offset makes the product read another sample. The reference's `process()` agrees with
    it everywhere for Tap; for TapLinear with fewer than 8 spare ring slots it reads samples of later lanes of its own 8-sample group
    (`tap_block`), which the product deliberately does not reproduce (DESIGN §10).

    Bound per output (first order; every rounding of the f32 form contributes U times the magnitude of its result, times the factor
    the later operations apply to it, all <= 3 since t <= 1): summing those over the Horner form of spline gives at most
    14.5|y0| + 38.5|y1| + 31|y2| + 7|y3| <= 39 S_t with S_t = sum_j |y_j|, and lerp's three roundings (b - a, * t, + a) at most 4 S_t.
    The N - 1 additions of the taps add at most N * 1.25 S_t each (|spline| <= 1.25 max|y_j|). So
      |f32 - f64| <= (39 + 2N) U sum_t S_t   (spline),   (4 + 2N) U sum_t S_t   (lerp).
    mutate: "offset" (every tap one sample later), "reverse" (spline taps in the order y3, y2, y1, y0), "round" (round(D) for floor(D))."""
    s, lo, hi, _ = tap_params(min_delay, max_delay, sr, linear)
    x = np.asarray(x, np.float64)
    n = x.size
    pad = int(hi * s) + 8
    h = np.concatenate([np.zeros(pad), x, np.zeros(2)])   # h[pad + k] = x[k]
    idx = np.arange(n) + pad
    y = np.zeros(n)
    S = np.zeros(n)
    delays = np.atleast_2d(np.asarray(delays, F32))
    for d in delays:
        D = tap_positions(d, lo, hi, s).astype(np.float64)
        f = np.floor(D + 0.5) if mutate == "round" else np.floor(D)
        if mutate == "offset":
            f = f + 1
        t = D - f
        f = f.astype(np.int64)
        y1, y2 = h[idx - f], h[idx - f - 1]
        if linear:
            y += y1 + (y2 - y1) * t
            S += np.abs(y1) + np.abs(y2)
        else:
            y0, y3 = h[idx - f + 1], h[idx - f - 2]
            if mutate == "reverse":
                y0, y1, y2, y3 = y3, y2, y1, y0
            y += y1 + t * 0.5 * (y2 - y0 + t * (2.0 * y0 - 5.0 * y1 + 4.0 * y2 - y3 + t * (3.0 * (y1 - y2) + y3 - y0)))
            S += np.abs(y0) + np.abs(y1) + np.abs(y2) + np.abs(y3)
    N = delays.shape[0]
    return y, ((4.0 if linear else 39.0) + 2.0 * N) * U * S


def tap_block(x, delays, min_delay, max_delay, sr, sizes, linear=False):
    """The reference's Tap / TapLinear `process()` as written, over the process() sizes `sizes`: each full 8-sample group first writes
    its 8 inputs into the power-of-two ring, then reads every lane at (i - (8 - k) - floor(D)) & mask (and its neighbours); the tail
    (size & 7) runs `tick`. Returns (y, aliased): y in f64, computed with the same expressions as `tap` above, and `aliased[n]` true where
    a lane read a ring slot that a LATER lane of its own group had already overwritten. That happens only when the ring has fewer than
    8 slots to spare behind the oldest sample a tap reads: never for Tap (the 1.00001-sample floor and the 3 + SIMD_N of headroom), but
    for TapLinear whenever floor(D) + 9 - k > ring, e.g. a ring of 2 (max = 0) or max * sr just under ring - 2. Where nothing aliases,
    y equals `tap`'s f64 value exactly: the block path and the tick path read the same samples."""
    s, lo, hi, ring = tap_params(min_delay, max_delay, sr, linear)
    mask = ring - 1
    x = np.asarray(x, np.float64)
    delays = np.atleast_2d(np.asarray(delays, F32))
    D = np.array([tap_positions(d, lo, hi, s).astype(np.float64) for d in delays])
    buf = np.zeros(ring)
    who = np.full(ring, -1, np.int64)   # which sample each slot holds (-1: the zero of a reset)
    y = np.zeros(x.size)
    aliased = np.zeros(x.size, bool)
    i = 0

    def read(n, pos):
        acc = 0.0
        for Dt in D[:, n]:
            f = int(np.floor(Dt))
            t = Dt - f
            slots = [(pos - f - j) & mask for j in ((0, 1) if linear else (-1, 0, 1, 2))]
            if any(who[sl] > n for sl in slots):
                aliased[n] = True
            v = [buf[sl] for sl in slots]
            if linear:
                acc += v[0] + (v[1] - v[0]) * t
            else:
                y0, y1, y2, y3 = v
                acc += y1 + t * 0.5 * (y2 - y0 + t * (2.0 * y0 - 5.0 * y1 + 4.0 * y2 - y3 + t * (3.0 * (y1 - y2) + y3 - y0)))
        y[n] = acc

    p = 0
    for m in sizes:
        for g in range(m >> 3):
            base = p + 8 * g
            for k in range(8):
                buf[i], who[i] = x[base + k], base + k
                i = (i + 1) & mask
            for k in range(8):
                read(base + k, (i - (8 - k)) & mask)
        for n in range(p + (m & ~7), p + m):
            buf[i], who[i] = x[n], n
            read(n, i)
            i = (i + 1) & mask
        p += m
    return y, aliased


# ---------------------------------------------------------------- FeedbackUnit (src/feedback.rs, ID 79)
def feedback_samples(delay_s, sr):
    """FeedbackUnit::set_sample_rate: samples = max(1, round(delay * sr)); the rings are next_power_of_two(samples) long."""
    return max(1, int(round_half_away(delay_s * sr)))


def feedback_block_mode(size, S):
    """FeedbackUnit::process takes the block path (the inner unit's own process() over the whole block) when size <= samples,
    and ticks the inner unit sample by sample otherwise."""
    return size <= S


def feedback_unit(x, delay_s, sr, gains, fir_w, mutate_s=0):
    """FeedbackUnit::new(delay, X) with a linear X per channel: X_c = g_c * pass() >> fir(w) for channel 0 (fir_w may be None:
    then X_0 = g_0 * pass()) and X_c = g_c * pass() for the others; fir(w) is y[n] = sum_i w[i] t[n - (K - 1 - i)] (src/fir.rs). x [channels][n]. With S = feedback_samples(delay, sr):
      u[n] = x[n] + y[n - S],   y = X(u)
    in f64 (y = 0 before the start). The block path reads y[n - S] of samples written before the block (size <= S) and the tick
    path reads it sample by sample, so both are this recurrence for a linear X.

    Bound (running, first order): the f32 form rounds u (U|u|), g * u (U|g u|) and the FIR (K products and K - 1 additions: at most
    K U sum_k |w_k t[n-k]|); the error of y[n - S] comes back through the loop multiplied by |g| sum_k |w_k| < 1, so it grows at most
    geometrically to 1 / (1 - |g| sum|w|) of the local rounding. The bound is carried along the recurrence:
      e_u[n] = e_y[n - S] + U|u[n]|,  e_t[n] = |g| e_u[n] + U|g u[n]|,  e_y[n] = sum_k |w_k| e_t[n-k] + K U sum_k |w_k t[n-k]|.
    mutate_s: S + mutate_s instead of S (a negative control)."""
    x = np.atleast_2d(np.asarray(x, np.float64))
    C, n = x.shape
    S = feedback_samples(delay_s, sr) + mutate_s
    y = np.zeros((C, n))
    e = np.zeros((C, n))
    for c in range(C):
        g = float(F32(gains[c]))
        # Fir::tick shifts its window v left and puts the new sample last: output = sum_i w[i] v[i], so the LAST weight multiplies t[n]
        w = np.asarray(fir_w if (c == 0 and fir_w is not None) else [1.0], F32).astype(np.float64)
        K = w.size
        t = np.zeros(n + K)
        et = np.zeros(n + K)
        for i in range(n):
            fb = y[c, i - S] if i >= S else 0.0
            efb = e[c, i - S] if i >= S else 0.0
            u = x[c, i] + fb
            ti = g * u
            t[i + K - 1] = ti
            et[i + K - 1] = abs(g) * (efb + U * abs(u)) + U * abs(ti)
            win, ewin = t[i: i + K], et[i: i + K]
            y[c, i] = float(np.dot(w, win))
            e[c, i] = float(np.dot(np.abs(w), ewin)) + (K * U * float(np.dot(np.abs(w), np.abs(win))) if K > 1 else 0.0)
    return y, e


# ---------------------------------------------------------------- Oversampler (src/oversample.rs, ID 51)
def halfband_min():
    """HALFBAND_MIN as the crate's [f32; 43] holds it (tests/golden/halfband_min.json, written by tests/golden/gen_halfband.py)."""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "halfband_min.json")) as f:
        bits = json.load(f)["f32_bits"]
    return np.array(bits, np.uint32).view(F32).astype(np.float64)


def _halfband_taps():
    """The reference's polyphase taps against the history, newest sample last. interpolating_filter reads the 24 ring slots
    newest - 23 ... newest (START_SAMPLE_OFFSET_HALF = 129 - 24) against INTERPOLATING_EVEN_COEFFS (two zeros, then h[0], h[2], ..., h[42])
    and INTERPOLATING_ODD_COEFFS (three zeros, then h[1], h[3], ..., h[41]), and doubles both sums; decimating_filter reads the 48 slots
    last - 47 ... last (START_SAMPLE_OFFSET_FULL = 129 - 48) against DECIMATING_COEFFS (five zeros, then h[0] ... h[42])."""
    h = halfband_min()
    ev = np.concatenate([[0.0, 0.0], h[0::2]])
    od = np.concatenate([[0.0, 0.0, 0.0], h[1::2]])
    dc = np.concatenate([np.zeros(5), h])
    return ev, od, dc


def oversample(x, sizes, gain=1.0, inner_delay=0, mutate=None):
    """Oversampler(X) over the process() sizes `sizes`, X = gain * pass() (inner_delay 0) or tick() * gain (inner_delay 1, which makes
    the zero the odd-size rule feeds inward visible). x: the outer input, at least sum(sizes) samples. Returns (y, bound).

    Oversampler::process(size) runs twice, over the halves [0, size/2) and [size/2, 2 (size/2)) (integer halves): each pushes its outer
    samples into the input ring and interpolates two inner samples from each, runs X's process(size) over the `size` inner samples of
    that half, and decimates every odd inner sample (the even one enters the output ring first). With an odd size the last outer
    sample is never read, its output is 0, and each half feeds X one zero inner sample (inner_input[size - 1] is never written)
    whose output is dropped. mutate (negative controls): "no_zero_feed" leaves that zero out; "stream" runs every size as one plain
    stream, as if the odd rule did not exist.

    Bound (first order): each interpolated sample is a sum of at most 21 products taken through eight lane accumulators and a
    three-level reduction, so every product sees at most 1 + 3 + 3 roundings: 7 U sum|h x| (the doubling is exact); the gain adds
    U|g v|; the decimated output is 48 lanes' worth (1 + 6 + 3 roundings): 10 U sum|h v| plus the inner errors carried through sum|h|."""
    ev, od, dc = _halfband_taps()
    g = float(F32(gain))
    xin, ein = [0.0] * 24, [0.0] * 24          # outer input history (zeros before the start)
    vin, evn = [0.0] * 48, [0.0] * 48          # inner output history, as the output ring receives it
    prev = [0.0, 0.0]                          # X's tick() state: value, bound
    x = np.asarray(x, np.float64)
    out, bound = [], []
    pos = 0

    def run_inner(u, eu):
        if inner_delay:
            v, e = prev[0], prev[1]
            prev[0], prev[1] = g * u, g * eu + (U * abs(g * u) if g != 1.0 else 0.0)
            return v, e
        return g * u, abs(g) * eu + (U * abs(g * u) if g != 1.0 else 0.0)

    def interp():
        a = np.array(xin[-24:])
        e = 2.0 * float(np.dot(ev, a)), 2.0 * float(np.dot(od, a))
        b = 2.0 * 7.0 * U * float(np.dot(np.abs(ev), np.abs(a))), 2.0 * 7.0 * U * float(np.dot(np.abs(od), np.abs(a)))
        return e, b

    def decim():
        a = np.array(vin[-48:])
        ea = np.array(evn[-48:])
        return float(np.dot(dc, a)), 10.0 * U * float(np.dot(np.abs(dc), np.abs(a))) + float(np.dot(np.abs(dc), ea))

    odd_rule = mutate != "stream"
    for size in sizes:
        halves = [(0, size // 2), (size // 2, size // 2)] if odd_rule else [(0, size)]
        for off, m in halves:
            inner = []
            for i in range(m):
                xin.append(float(x[pos + off + i]))
                (e0, e1), (b0, b1) = interp()
                inner += [(e0, b0), (e1, b1)]
            inner_out = [run_inner(u, b) for u, b in inner]
            if odd_rule and size % 2 and mutate != "no_zero_feed":
                run_inner(0.0, 0.0)   # inner_input[size - 1]: the zero each half feeds X
            for i in range(m):
                for k in (0, 1):
                    vin.append(inner_out[2 * i + k][0]); evn.append(inner_out[2 * i + k][1])
                v, b = decim()
                out.append(v); bound.append(b)
        if odd_rule and size % 2:
            out.append(0.0); bound.append(0.0)
        pos += size
    return np.array(out), np.array(bound)
