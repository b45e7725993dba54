"""Deterministic synthetic PCM for the golden cases: a few sines per channel + noise, as float32 ring contents in
(-0.5, 0.5) like fifo.c's s16 / 65535 (fifo.c:104-107).  Built from PCG64 bit streams only (stable across numpy
versions); the goldens carry a checksum of what the generating run used."""
import numpy as np


def pcm_frames(seed, n, frames, hop=None):
    """-> (lb [frames][n], rb [frames][n]) float32: ring contents of `frames` consecutive updates, sliding by `hop`"""
    hop = hop or max(n // 16, 64)
    total = n + hop * frames
    rng = np.random.Generator(np.random.PCG64(seed))
    t = np.arange(total, dtype=np.float64)
    out = []
    for ch in range(2):
        k = 3 + int(rng.integers(0, 4))
        freqs = rng.integers(2, n // 8, size=k).astype(np.float64) / n
        amps = (rng.integers(60, 420, size=k).astype(np.float64) / 1000.0) * (0.6 if ch else 1.0)
        sig = sum(a * np.sin(2 * np.pi * f * t + ch) for a, f in zip(amps, freqs))
        env = 0.4 + 0.6 * np.abs(np.sin(2 * np.pi * t / (hop * 3.7)))
        noise = rng.integers(-9000, 9000, size=total).astype(np.float64) / 65535.0
        s16 = np.clip(np.round((sig * env + noise) * 32767.0 * 0.5), -32768, 32767).astype(np.int16)
        out.append(s16.astype(np.float32) / np.float32(65535))
    lb = np.stack([out[0][(i + 1) * hop:(i + 1) * hop + n] for i in range(frames)])
    rb = np.stack([out[1][(i + 1) * hop:(i + 1) * hop + n] for i in range(frames)])
    return np.ascontiguousarray(lb), np.ascontiguousarray(rb)


def checksum(a):
    return int(np.frombuffer(np.ascontiguousarray(a).tobytes(), np.uint8).astype(np.uint64).sum())


EDGE_SIGNALS = ["noise", "silence", "dc", "nyquist", "impulse_first", "impulse_last", "tone_on_bin", "tone_half_bin",
                "square", "noise_1e-4", "tone_plus_1e-5"]


def edge_signal(kind, n):
    """float32 PCM in [-0.5, 0.5] where FFT indexing and twiddle bugs show.  The transform is the packed (n/2)-point
    complex FFT of z[k] = x[2k] + i x[2k+1]: a tone of b / n cycles per sample is b / (n/2) cycles per complex point,
    on bin b of it for a whole b and half a bin off for b + 0.5."""
    i = np.arange(n, dtype=np.float64)
    rng = np.random.default_rng(n + EDGE_SIGNALS.index(kind))
    tone = lambda b: 0.45 * np.cos(2 * np.pi * b * i / n)
    x = {"noise": lambda: np.clip(rng.standard_normal(n) * 0.2, -0.5, 0.5),
         "silence": lambda: np.zeros(n),
         "dc": lambda: np.full(n, 0.37),
         "nyquist": lambda: np.where(i % 2 == 0, 0.5, -0.5),
         "impulse_first": lambda: np.where(i == 0, 0.5, 0.0),
         "impulse_last": lambda: np.where(i == n - 1, -0.5, 0.0),
         "tone_on_bin": lambda: tone(n // 16),
         "tone_half_bin": lambda: tone(n // 16 + 0.5),
         "square": lambda: np.where((i // (n // 8)) % 2 == 0, 0.5, -0.5),
         "noise_1e-4": lambda: rng.standard_normal(n) * 1e-4,
         "tone_plus_1e-5": lambda: tone(n // 16 + 0.5) + rng.standard_normal(n) * 1e-5}[kind]()
    return x.astype(np.float32)


def fft_ramp(n, fft_scale=10.2, fft_cutoff=0.3):
    """render.c:845's per-bin gain max(i / sz * fft_scale + 1 - fft_cutoff, 1), float parameters, evaluated in float64"""
    return np.maximum(np.arange(n) / n * np.float64(np.float32(fft_scale)) + (1.0 - np.float64(np.float32(fft_cutoff))), 1.0)


def fft_magnitude_error(got, f64):
    """transform_fft output (log(|X| + 1) / 3 * ramp) -> max error of |X| over the peak |X|, against the float64 evaluation.

    Measured on |X| rather than on the output: the log compresses a concentrated spectrum's peak (DC, a pure tone: |X| in the
    hundreds, output ~20) while a float32 FFT's absolute error follows the signal's energy, so "of peak output" is no bound on
    the transform there.  Discounted per bin: the reference's own float rounding of |X| + 1 (render.c:844, up to 2^-24 of it)
    and of the float output (ln(|X| + 1) * 2^-24 of |X| + 1) — render.c's arithmetic, kept by the kernels."""
    r = fft_ramp(got.shape[0])
    v_got = np.expm1(3 * np.asarray(got, np.float64) / r); v = np.expm1(3 * np.asarray(f64, np.float64) / r)
    floor = (v + 1) * 2.0 ** -24 * (1 + np.log1p(v))
    return np.maximum(np.abs(v_got - v) - floor, 0).max() / v.max()
