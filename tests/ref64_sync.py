"""Float64 reference of the cell search, written from 36.211 6.11 and DESIGN.md §2 ("cell search") with numpy only: the PSS / SSS sequences, a
synthesiser of sync-only captures for symbol sizes the simulator does not cover (N = 128: 6 PRB), and the search's metrics, CFO sum and SSS table."""
import numpy as np

ROOTS = (25, 29, 34)
BINS = 9600


def pss(n_id_2):
    """d_u(n), n = 0..61 (36.211 6.11.1.1)"""
    u = ROOTS[n_id_2]
    n = np.arange(62)
    m = np.where(n < 31, n * (n + 1), (n + 1) * (n + 2))
    return np.exp(-1j * np.pi * u * m / 63)


def _mseq(taps):
    x = [0, 0, 0, 0, 1]
    while len(x) < 31:
        x.append(sum(x[len(x) - 5 + t] for t in taps) % 2)
    return 1 - 2 * np.array(x)


S_T, C_T, Z_T = _mseq([2, 0]), _mseq([3, 0]), _mseq([4, 2, 1, 0])   # x(i+5) = x(i+2)+x(i), x(i+3)+x(i), x(i+4)+x(i+2)+x(i+1)+x(i)


def sss(n_id_1, n_id_2, sf5):
    """d(n), n = 0..61, of subframe 0 (sf5 = 0) or 5 (36.211 6.11.2.1)"""
    qp = n_id_1 // 30
    q = (n_id_1 + qp * (qp + 1) // 2) // 30
    mp = n_id_1 + q * (q + 1) // 2
    m0 = mp % 31
    m1 = (m0 + mp // 31 + 1) % 31
    n = np.arange(31)
    s0, s1 = S_T[(n + m0) % 31], S_T[(n + m1) % 31]
    c0, c1 = C_T[(n + n_id_2) % 31], C_T[(n + n_id_2 + 3) % 31]
    z0, z1 = Z_T[(n + m0 % 8) % 31], Z_T[(n + m1 % 8) % 31]
    d = np.zeros(62)
    d[0::2] = s1 * c0 if sf5 else s0 * c0
    d[1::2] = s0 * c1 * z1 if sf5 else s1 * c1 * z0
    return d


def subcarriers():
    """frequency index of d(n): -31..-1, 1..31"""
    n = np.arange(62)
    return np.where(n < 31, n - 31, n - 30)


def synth(N, pci, nsf, rng, t0=0, nsc=72):
    """nsf subframes (first = subframe t0) of one antenna: PSS / SSS in subframes 0 and 5, unit-power QPSK on every other RE of the nsc sub-carriers"""
    f = subcarriers()
    out = []
    for i in range(nsf):
        sf = (t0 + i) % 10
        for l in range(14):
            X = np.zeros(N, complex)
            k = np.concatenate([np.arange(-nsc // 2, 0), np.arange(1, nsc // 2 + 1)])
            X[k % N] = (rng.choice([-1, 1], len(k)) + 1j * rng.choice([-1, 1], len(k))) / np.sqrt(2)
            if sf in (0, 5) and l in (5, 6):
                X[f % N] = pss(pci % 3) if l == 6 else sss(pci // 3, pci % 3, sf == 5)
            x = np.fft.ifft(X) * np.sqrt(N)
            cp = (160 if l % 7 == 0 else 144) * N // 2048
            out.append(np.concatenate([x[-cp:], x]))
    return np.concatenate(out)


def replicas(N):
    """p_u[k] = (1/sqrt N) sum_n d_u(n) exp(+j 2 pi f_n k / N)"""
    k = np.arange(N)
    return np.array([(pss(u)[:, None] * np.exp(2j * np.pi * subcarriers()[:, None] * k[None, :] / N)).sum(0) / np.sqrt(N) for u in range(3)])


def metric(x, t, p):
    """sum_a |c_a|^2 / (E_p sum_a E_a) of the windows starting at the samples t (array)"""
    N = len(p)
    idx = np.asarray(t)[:, None] + np.arange(N)[None, :]
    P = sum(np.abs((xa[idx] * np.conj(p)).sum(1)) ** 2 for xa in x)
    E = sum((np.abs(xa[idx]) ** 2).sum(1) for xa in x)
    return P / ((np.abs(p) ** 2).sum() * E)


def search(N, x, taus=None):
    """float64 restatement of the search: coarse fold [3][9600], refined [3][2D-1] and, at the timing taus[u] (default: this function's own),
    the CFO sum S[u] and the SSS table [3][168][2]"""
    x = np.asarray(x, complex)
    L, D, HF = x.shape[1], N // 128, 75 * N
    J = (L - N) // D + 1
    rep = replicas(N)
    coarse, refined, S, tab, tau_out = np.zeros((3, BINS)), np.zeros((3, 2 * D - 1)), np.zeros(3, complex), np.zeros((3, 168, 2)), []
    f = subcarriers()
    for u in range(3):
        m = metric(x, np.arange(J) * D, rep[u])
        for b in range(BINS):
            coarse[u, b] = m[b::BINS].mean()
        bp = int(np.argmax(coarse[u]))
        for i in range(2 * D - 1):
            t0 = (bp * D + HF + i - (D - 1)) % HF
            refined[u, i] = metric(x, np.arange(t0, L - N + 1, HF), rep[u]).mean()
        tau = (bp * D + HF + int(np.argmax(refined[u])) - (D - 1)) % HF if taus is None else taus[u]
        tau_out.append(tau)
        k = np.arange(N)
        for h, t in enumerate(range(tau, L - N + 1, HF)):
            for xa in x:
                c1 = (xa[t:t + N // 2] * np.conj(rep[u][:N // 2])).sum()
                c2 = (xa[t + N // 2:t + N] * np.conj(rep[u][N // 2:])).sum()
                S[u] += c2 * np.conj(c1)
        cfo = np.angle(S[u]) * 15000 / np.pi
        rot = np.exp(-2j * np.pi * cfo * (N + 9 * D) / (15000 * N))
        Wf = np.exp(-2j * np.pi * f[:, None] * k[None, :] / N)
        s_all = np.array([[sss(n1, u, q) for q in (0, 1)] for n1 in range(168)])
        for h, t in enumerate(range(tau, L - N + 1, HF)):
            if t < N + 9 * D:
                continue
            z = sum((Wf @ xa[t - N - 9 * D:t - 9 * D]) * np.conj((Wf @ xa[t:t + N]) * np.conj(pss(u)) * rot) for xa in x)
            a = s_all @ z.real                     # [168][2]: correlation with the sf-0 / sf-5 sequence
            tab[u] += a if h % 2 == 0 else a[:, ::-1]
    return dict(coarse=coarse, refined=refined, S=S, sss=tab, tau=tau_out)
