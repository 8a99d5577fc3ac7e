"""Float64 reference of the tracker, written from DESIGN.md §2 ("tracking") with numpy only: the cell search's stride-1 metric over each
half-frame's window, the argmax with its tie order, the CFO sum S, and the timing / carrier-offset rule.  Returns what the oracle's records say."""
import numpy as np

import ref64_sync as R

P, ALPHA, MISS, LOCK_K = 4, 0.05, 4, 20.0


def track(N, x, pci, frame_offset, cfo_hz, first_tti=0, no_cfo=False, max_sf=10 ** 9):
    """x complex [A][L] from absolute sample 0 -> dict of arrays: start, tti, flags (per subframe), delta, peak, S, locked (per half-frame)"""
    x = np.asarray(x, complex)
    L, SF, W = x.shape[1], 15 * N, 9 * N // 128
    p = R.replicas(N)[pci % 3]
    s, k, f, d, acc = frame_offset, 0, float(cfo_hz), 0.0, 0.0
    miss = nhf = ncor = 0
    lk = []                       # (h, delta) of the locked half-frames since the last correction
    out = dict(start=[], flags=[], cfo=[], delta=[], peak=[], S=[], locked=[])
    order = [0] + [sg * m for m in range(1, W + 1) for sg in (-1, 1)]
    while k < max_sf and s + SF <= L:
        tti = (first_tti + k) % 10240
        out["start"].append(s), out["cfo"].append(f)
        out["flags"].append((1 if miss == 0 else 0) | (2 if miss >= MISS else 0))
        if tti % 5 == 0:
            tau = s + 13 * N // 2
            m = R.metric(x, tau + np.array(order), p)
            i = int(np.argmax(m))             # first maximum in the order 0, -1, +1, -2, ...
            delta, peak = order[i], m[i]
            t = tau + delta
            Sv = sum((xa[t + N // 2:t + N] * np.conj(p[N // 2:])).sum() * np.conj((xa[t:t + N // 2] * np.conj(p[:N // 2])).sum()) for xa in x)
            hn = nhf
            nhf += 1
            locked = peak >= LOCK_K / N
            out["delta"].append(delta), out["peak"].append(peak), out["S"].append(Sv), out["locked"].append(locked)
            if locked:
                miss = 0
                if not no_cfo:
                    f = f + ALPHA * (np.angle(Sv) * 15000 / np.pi - f)
                lk.append((hn, delta))
                if len(lk) == P:
                    sd = sum(v for _, v in lk)
                    c = int(np.sign(sd)) * ((abs(sd) + P // 2) // P)
                    s += c
                    ncor += 1
                    if ncor == 1:
                        h = np.array([a for a, _ in lk], float)
                        v = np.array([b for _, b in lk], float)
                        d = d + np.polyfit(h, v, 1)[0]
                    else:
                        d = (s - frame_offset - k * SF) / (nhf - 0.5 * (P - 1))
                    lk = []
            else:
                miss += 1
        acc += d / 5
        r = np.floor(abs(acc) + 0.5) * np.sign(acc)     # half away from zero, as roundf
        acc -= r
        s += SF + int(r)
        k += 1
    return {key: np.array(v) for key, v in out.items()}
