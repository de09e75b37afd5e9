"""TEST INFRASTRUCTURE ONLY -- numpy model of the FFT decomposition used by the CUDA kernels.

Not part of the product path: only tests/ may import this file.  It restates, in
vectorised numpy, the exact algebra the sm_90a kernels in
``hyena-dna_b200/csrc/`` implement, so the index bookkeeping (4-step layout, row
pairing, even/odd polyphase pointwise product, scaling) can be checked on a CPU
against ``numpy.fft`` before any GPU time is spent.

What it models (reference semantics: src/models/sequence/hyena.py:59-88 fftconv_ref,
standalone_hyenadna.py:45-60):

  y[t] = sum_{j<=t} k[j] g[t-j],   t in [0, L)          (causal linear convolution)

computed as a length n = 2*M real FFT convolution (n >= 2L, M = M1*M2 a power of two)
through ONE complex FFT of length M on the packed signal z[m] = x[2m] + i x[2m+1].

Layout: the length-M complex FFT is split Cooley-Tukey style with m = M2*m1 + m2 and
k = k1 + M1*k2.  Spectra live in "[k1][k2]" order, i.e. element (k1, k2) holds bin
k = k1 + M1*k2.  Bin k pairs with bin M-k, which lives at row (M1-k1)%M1 and column
(M2 - k2 - (k1 != 0)) % M2.
"""
import numpy as np


def pack_real(x, M):
    """x: real (..., <=2M) -> complex (..., M): z[m] = x[2m] + i x[2m+1], zero padded."""
    buf = np.zeros(x.shape[:-1] + (2 * M,), dtype=np.float64)
    buf[..., : x.shape[-1]] = x
    return buf[..., 0::2] + 1j * buf[..., 1::2]


def four_step_fwd(z, M1, M2):
    """Pass 1 (column FFT over m1 + twiddle) and pass 2a (row FFT over m2).

    z: (..., M) natural order -> Z: (..., M1, M2) with Z[k1, k2] = FFT_M(z)[k1 + M1*k2].
    """
    M = M1 * M2
    a = z.reshape(z.shape[:-1] + (M1, M2))             # a[m1, m2] = z[M2*m1 + m2]
    A = np.fft.fft(a, axis=-2)                          # over m1 -> k1
    k1 = np.arange(M1)[:, None]
    m2 = np.arange(M2)[None, :]
    A = A * np.exp(-2j * np.pi * (k1 * m2) / M)         # W_M^{m2 k1}
    return np.fft.fft(A, axis=-1)                       # over m2 -> k2


def four_step_inv(Zp, M1, M2):
    """Pass 2b (inverse row FFT + conj twiddle) and pass 3 (inverse column FFT); UNSCALED.

    Zp: (..., M1, M2) in [k1][k2] order -> z': (..., M) natural order, z' = M * ifft(Z').
    """
    M = M1 * M2
    A = np.fft.ifft(Zp, axis=-1) * M2                   # over k2 -> m2, unscaled
    k1 = np.arange(M1)[:, None]
    m2 = np.arange(M2)[None, :]
    A = A * np.exp(+2j * np.pi * (k1 * m2) / M)
    a = np.fft.ifft(A, axis=-2) * M1                    # over k1 -> m1, unscaled
    return a.reshape(a.shape[:-2] + (M,))


def partner(Z, M1, M2):
    """P[k1,k2] = Z at bin M-k (the kernels fetch this through shared memory)."""
    k1 = np.arange(M1)
    k2 = np.arange(M2)
    pr = (M1 - k1) % M1
    pc = (M2 - k2[None, :] - (k1[:, None] != 0)) % M2
    return Z[..., pr[:, None], pc]


def wk(M1, M2):
    """W_M^k at [k1][k2]."""
    M = M1 * M2
    k = np.arange(M1)[:, None] + M1 * np.arange(M2)[None, :]
    return np.exp(-2j * np.pi * k / M)


def eo(Z, M1, M2):
    """2x the even/odd-sample spectra: E2 = Z + conj(P), O2 = -i (Z - conj(P))."""
    P = np.conj(partner(Z, M1, M2))
    return Z + P, -1j * (Z - P)


def pointwise_conv(Zg, Zk, M1, M2):
    """Forward product: spectrum (packed form) of the convolution, times 4."""
    E, O = eo(Zg, M1, M2)
    He, Ho = eo(Zk, M1, M2)
    W = wk(M1, M2)
    Ye = E * He + W * O * Ho
    Yo = E * Ho + O * He
    return Ye + 1j * Yo


def pointwise_corr(Zd, Zh, M1, M2):
    """Backward product: packed spectrum of corr(d, h)[j] = sum_t d[t] h[t-j], times 4.

    Used for dg (h = filter k) and for dk (h = gated input g).
    """
    E, O = eo(Zd, M1, M2)
    He, Ho = eo(Zh, M1, M2)
    W = wk(M1, M2)
    Ye = E * np.conj(He) + O * np.conj(Ho)
    Yo = np.conj(W) * E * np.conj(Ho) + O * np.conj(He)
    return Ye + 1j * Yo


def unpack_real(zp, L):
    out = np.empty(zp.shape[:-1] + (2 * zp.shape[-1],))
    out[..., 0::2] = zp.real
    out[..., 1::2] = zp.imag
    return out[..., :L]


def causal_conv(g, k, M1, M2):
    M = M1 * M2
    L = g.shape[-1]
    Zg = four_step_fwd(pack_real(g, M), M1, M2)
    Zk = four_step_fwd(pack_real(k, M), M1, M2)
    zp = four_step_inv(pointwise_conv(Zg, Zk, M1, M2), M1, M2)
    return unpack_real(zp, L) / (4.0 * M)


def causal_corr(d, h, M1, M2):
    M = M1 * M2
    L = d.shape[-1]
    Zd = four_step_fwd(pack_real(d, M), M1, M2)
    Zh = four_step_fwd(pack_real(h, M), M1, M2)
    zp = four_step_inv(pointwise_corr(Zd, Zh, M1, M2), M1, M2)
    return unpack_real(zp, L) / (4.0 * M)


# ---------------------------------------------------------------------------
# two-stage in-block FFT exactly as the kernels schedule it (radix R1 then R2)
# ---------------------------------------------------------------------------
def block_fft_two_stage(x, R1, R2, inverse=False):
    """N = R1*R2 point FFT the way a thread group does it.

    stage 1: thread n2 in [0,R2) takes x[R2*n1 + n2], n1 in [0,R1) -> radix-R1 FFT -> k1'
             multiplies by W_N^{n2 k1'} and writes exchange[k1'][n2]
    stage 2: work item k1' reads exchange[k1'][0..R2) -> radix-R2 FFT -> X[k1' + R1*k2']
    """
    N = R1 * R2
    sgn = +1.0 if inverse else -1.0
    a = x.reshape(x.shape[:-1] + (R1, R2))
    f = (lambda v, ax: np.fft.ifft(v, axis=ax) * v.shape[ax]) if inverse else (lambda v, ax: np.fft.fft(v, axis=ax))
    s1 = f(a, -2)
    k1p = np.arange(R1)[:, None]
    n2 = np.arange(R2)[None, :]
    s1 = s1 * np.exp(sgn * 2j * np.pi * (k1p * n2) / N)
    s2 = f(s1, -1)                                      # [k1'][k2']
    out = np.empty(x.shape, dtype=complex)
    k = (np.arange(R1)[:, None] + R1 * np.arange(R2)[None, :]).reshape(-1)
    out[..., k] = s2.reshape(s2.shape[:-2] + (N,))
    return out
