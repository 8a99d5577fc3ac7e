"""Float64 reference of the tracker with its find state (LTEPHY_TRACK_REACQUIRE), written from DESIGN.md §2 ("tracking", "cell search") with
numpy only: ref64_track's timing rule, and after 4 half-frames in a row without lock the cell search of ref64_sync.search on one frame plus a
symbol at a time, its detection rule and frame timing restated from the search's tables.  Returns what the oracle's subframe records say."""
import numpy as np

import ref64_sync as R
from ref64_track import ALPHA, LOCK_K, MISS, P

PSR_MIN, SSS_MIN = 2.5, 1.75


def find(N, w, pci):
    """the cell search's result for N_ID_2 = pci mod 3 on the window w [A][150 N + N] -> (detected with this pci, frame_offset, cfo_hz)"""
    u, HF, FR = pci % 3, 75 * N, 150 * N
    t = R.search(N, w)
    fold = t["coarse"][u]
    bp = int(np.argmax(fold))
    d = np.abs(np.arange(len(fold)) - bp)
    side = fold[np.minimum(d, len(fold) - d) > 2].max()
    psr = fold[bp] / side if side > 0 else np.inf
    a = t["sss"][u].reshape(-1)                      # [N_ID_1][q] flattened: index 2 N_ID_1 + q
    best = int(np.argmax(a))
    second = np.delete(a, best).max()
    ratio = a[best] / second if second > 0 else np.inf
    st = t["tau"][u] - 13 * N // 2
    fo = (st - (HF if best & 1 else 0)) % FR
    found = psr >= PSR_MIN and ratio >= SSS_MIN and 3 * (best // 2) + u == pci
    return found, int(fo), float(np.angle(t["S"][u]) * 15000 / np.pi)


def track(N, x, pci, frame_offset, cfo_hz, first_tti=0, no_cfo=False):
    """x complex [A][L] from absolute sample 0 -> dict of arrays per subframe: start, tti, flags (LOCKED 1, LOST 2, REACQUIRED 4); and finds"""
    x = np.asarray(x, complex)
    L, SF, W, FR = x.shape[1], 15 * N, 9 * N // 128, 150 * N
    p = R.replicas(N)[pci % 3]
    s, k, f, d, acc, base = frame_offset, 0, float(cfo_hz), 0.0, 0.0, frame_offset
    miss = nhf = ncor = finds = 0
    lk, searching, reacq, f0, kn = [], False, False, 0, 0
    out = dict(start=[], tti=[], flags=[])
    order = [0] + [sg * m for m in range(1, W + 1) for sg in (-1, 1)]
    while True:
        if searching:
            if f0 + FR + N > L:
                break
            finds += 1
            ok, fo, cfo = find(N, x[:, f0:f0 + FR + N], pci)
            if not ok:
                f0, kn = f0 + FR, kn + 10
                continue
            s, k = f0 + fo % SF, kn + ((10 - fo // SF) % 10 - (first_tti + kn)) % 10
            f = f if no_cfo else cfo
            miss, acc, lk, ncor, base, nhf = 0, 0.0, [], 0, s - k * SF, 0
            searching, reacq = False, True
            continue
        if s + SF > L:
            break
        tti = (first_tti + k) % 10240
        out["start"].append(s), out["tti"].append(tti)
        out["flags"].append((1 if miss == 0 else 0) | (2 if miss >= MISS else 0) | (4 if reacq else 0))
        reacq, lost_now = False, False
        if tti % 5 == 0:
            tau = s + 13 * N // 2
            m = R.metric(x, tau + np.array(order), p)
            i = int(np.argmax(m))
            delta = order[i]
            hn = nhf
            nhf += 1
            if m[i] >= LOCK_K / N:
                miss = 0
                if not no_cfo:
                    t = tau + delta
                    Sv = sum((xa[t + N // 2:t + N] * np.conj(p[N // 2:])).sum() * np.conj((xa[t:t + N // 2] * np.conj(p[:N // 2])).sum()) for xa in x)
                    f = f + ALPHA * (np.angle(Sv) * 15000 / np.pi - f)
                lk.append((hn, delta))
                if len(lk) == P:
                    sd = sum(v for _, v in lk)
                    s += int(np.sign(sd)) * ((abs(sd) + P // 2) // P)
                    ncor += 1
                    if ncor == 1:
                        d = d + np.polyfit(np.array([a for a, _ in lk], float), np.array([b for _, b in lk], float), 1)[0]
                    else:
                        d = (s - base - k * SF) / (nhf - 0.5 * (P - 1))
                    lk = []
            else:
                miss += 1
                lost_now = miss == MISS
        acc += d / 5
        r = np.floor(abs(acc) + 0.5) * np.sign(acc)     # half away from zero, as roundf
        acc -= r
        s += SF + int(r)
        k += 1
        if lost_now:
            searching, f0, kn = True, s, k
    return dict(start=np.array(out["start"]), tti=np.array(out["tti"]), flags=np.array(out["flags"]), finds=finds)
