"""NumPy restatement of truncated sampling (bagel_sample_rows_filtered_bf16), independent of the product: the top-k,
top-p and min-p thresholds of one row (fp64 mass, the fp32 min-p expression) and the Gumbel-max draw among the logits
at or above their maximum, with the Philox uniforms of sampling_oracle."""
import numpy as np

from sampling_oracle import gumbel_scores


def _f32(x):
    return np.asarray(x, dtype=np.float32)


def thresholds(row, inv_t, top_k=None, top_p=None, min_p=None, eps=0.0):
    """Candidate thresholds (tau_k, tau_p, tau_min) of one row of bf16-valued logits; -inf where a filter is off or the
    row has no finite logit. tau_p and tau_min are sets: the exact threshold and, with eps > 0, a neighbouring one where
    the top-p mass lies within relative eps of top_p * total, or where the fp32 min-p test of some logit moves when
    log(min_p) moves by up to 2 ulps (an fp32 sum or log may fall on either side there)."""
    l = np.asarray(row, dtype=np.float64)
    fin = l[np.isfinite(l)]
    if fin.size == 0:
        return -np.inf, {-np.inf}, {-np.inf}
    lmax = fin.max()
    tau_k = -np.inf
    if top_k and top_k < fin.size:
        tau_k = np.sort(fin)[::-1][top_k - 1]
    kept = fin[fin >= tau_k]
    tau_p = {-np.inf}
    if top_p is not None and top_p < 1.0:
        vals, inv = np.unique(kept, return_inverse=True)           # ascending distinct values
        e = np.exp((kept - lmax) * float(_f32(inv_t)))
        mass = np.bincount(inv, weights=e, minlength=vals.size)[::-1]   # per distinct value, descending
        vals = vals[::-1]
        cum = np.cumsum(mass)
        target = top_p * cum[-1]
        i = int(np.argmax(cum >= target))
        tau_p = {vals[i]}
        if i > 0 and cum[i - 1] >= target * (1 - eps):
            tau_p.add(vals[i - 1])
        if i + 1 < vals.size and cum[i] < target * (1 + eps):
            tau_p.add(vals[i + 1])
    tau_min = {-np.inf}
    if min_p:
        x = (_f32(fin) - _f32(lmax)) * _f32(inv_t)
        lmp = _f32(np.log(np.float32(min_p)))
        tau_min = {fin[x >= lmp].min()}
        if eps:
            for direction in (-np.inf, np.inf):
                t = lmp
                for _ in range(2):
                    t = np.nextafter(t, np.float32(direction), dtype=np.float32)
                    if (x >= t).any():
                        tau_min.add(fin[x >= t].min())
    return tau_k, tau_p, tau_min


def floors(row, inv_t, top_k=None, top_p=None, min_p=None, eps=0.0):
    """Every floor max(tau_k, tau_p, tau_min) the candidate thresholds allow, the exact one first."""
    tk, (tp,), (tm,) = thresholds(row, inv_t, top_k, top_p, min_p)
    exact = max(tk, tp, tm)
    _, tps, tms = thresholds(row, inv_t, top_k, top_p, min_p, eps)
    return [exact] + sorted({max(tk, p, m) for p in tps for m in tms} - {exact})


def kept(row, floor):
    l = np.asarray(row, dtype=np.float64)
    return np.isfinite(l) & (l >= floor)


def draw(row, temperature, key64, step, floor):
    """(token, decided) of the Gumbel-max draw among the logits >= floor: decided is False where the two best fp64
    scores lie within 1e-5 (fp32 scores may order them either way). An all-NaN row gives token 0."""
    keep = kept(row, floor)
    if not keep.any():
        return 0, True
    s = gumbel_scores(np.where(keep, row, 0.0), temperature, key64, step)
    s = np.where(keep, s, -np.inf)
    top2 = np.sort(s)[-2:]
    return int(np.argmax(s)), bool(top2[1] - top2[0] > 1e-5 * max(1.0, abs(top2[1])))


def truncated_softmax(row, temperature, floor):
    """fp64 probabilities of the truncated, renormalised softmax(l / T)."""
    l = np.asarray(row, dtype=np.float64)
    keep = kept(row, floor)
    z = np.where(keep, l / temperature, -np.inf)
    p = np.exp(z - z[keep].max())
    return p / p.sum()
