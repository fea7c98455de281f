"""Closed-form IMU-like streams for the spline-error-weighting tests (tests/test_sew_spectrum.py) and their fixtures
(tests/golden/make_sew_golden.py).  Every stream is a deterministic function of its length, so inputs of any size are regenerated
instead of committed; only the reference's outputs are stored."""
import numpy as np

RATE = 400.0                    # Hz
KINDS = ("tones", "gravity", "jitter")


def tones(n):
    """Incommensurate tones on all three axes, plus a bin-exact cosine at k = n // 3 and the alternating (Nyquist) sequence."""
    i = np.arange(n, dtype=np.float64)
    t = i / RATE
    k3 = n // 3
    x = np.empty((n, 3))
    x[:, 0] = 0.7 * np.sin(2 * np.pi * np.sqrt(2.0) * t + 0.3) + 0.2 * np.cos(2 * np.pi * 17.0 * np.pi * t) + 0.05 * np.cos(2 * np.pi * k3 * i / n)
    x[:, 1] = 0.4 * np.cos(2 * np.pi * (1 + np.sqrt(5.0)) / 2 * 3.1 * t) + 0.1 * (1.0 - 2.0 * (np.arange(n) % 2)) + 0.03
    x[:, 2] = 0.25 * np.sin(2 * np.pi * np.e * 11.0 * t - 1.1) + 0.05 * np.cos(2 * np.pi * k3 * i / n + 0.4) - 0.02
    return t, x


def gravity(n):
    """A resting accelerometer: 9.81 m/s2 of DC on z plus milli-g vibration and a slow sway on every axis."""
    t = np.arange(n, dtype=np.float64) / RATE
    x = np.empty((n, 3))
    x[:, 0] = 0.012 * np.sin(2 * np.pi * 37.3 * t) + 0.004 * np.sin(2 * np.pi * 0.21 * t + 0.5)
    x[:, 1] = -0.02 + 0.009 * np.cos(2 * np.pi * 52.9 * t + 1.0) + 0.003 * np.sin(2 * np.pi * 113.7 * t)
    x[:, 2] = 9.81 + 0.015 * np.sin(2 * np.pi * 24.1 * t + 2.0) + 0.002 * np.cos(2 * np.pi * 0.37 * t)
    return t, x


def jitter(n):
    """A gyroscope on a jittered clock with one sample dropped: n samples of a band-limited rotation rate at the actual times."""
    i = np.arange(n + 1, dtype=np.float64)
    t = (i + 0.02 * np.sin(1.618033988749895 * i) + 0.015 * np.sin(0.7548776662466927 * i * i % 6.283185307179586)) / RATE
    t = np.delete(t, (n + 1) // 2)
    x = np.empty((n, 3))
    x[:, 0] = 0.9 * np.sin(2 * np.pi * 0.83 * t) + 0.3 * np.sin(2 * np.pi * 4.7 * t + 0.2)
    x[:, 1] = 0.6 * np.cos(2 * np.pi * 1.37 * t + 0.9) + 0.15 * np.sin(2 * np.pi * 9.1 * t)
    x[:, 2] = -0.4 * np.sin(2 * np.pi * 2.11 * t + 0.4) + 0.05 * np.cos(2 * np.pi * 31.0 * t) + 0.01
    return t, x


def make(kind, n):
    """(times (n,), signal (n, 3)) of one of KINDS."""
    return {"tones": tones, "gravity": gravity, "jitter": jitter}[kind](n)


def reference_spectrum(x):
    """python/sew.py:make_reference_spectrum on an (n, 3) stream: Xhat_k = sqrt(1/3 sum_ch |FFT(x_ch)_k|^2), Xhat_0 = 0."""
    S = np.fft.fft(np.asarray(x, dtype=np.float64).T, axis=1)
    S[:, 0] = 0
    return np.sqrt(1.0 / 3.0) * np.linalg.norm(S, axis=0)


def spline_response(freqs, dt):
    """python/sew.py:spline_interpolation_response: 3 sinc(f dt)^4 / (2 + cos(2 pi f dt)), normalised at f = 0."""
    y = np.asarray(freqs, dtype=np.float64) * dt
    return 3.0 * np.sinc(y) ** 4 / (2.0 + np.cos(2.0 * np.pi * y))
