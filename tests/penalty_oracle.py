"""NumPy oracle of the decode-step penalties (bagel_apply_penalties_bf16, include/bagel_b200.h): with c_t the number of
times token t occurs in the tokens a request has generated, every bf16 logit l_t with c_t > 0 becomes
bf16_rne(((l < 0 ? l * rp : l / rp) - fp * c_t) - pp), in fp32 with one rounding per operation. Other logits, NaN
logits (bits kept) and rows with every penalty off are unchanged. No product code."""
import numpy as np
import torch


def is_off(rp=1.0, fp=0.0, pp=0.0):
    """The row is untouched: the fp32 values equal the off values."""
    return np.float32(rp) == 1 and np.float32(fp) == 0 and np.float32(pp) == 0


def apply(row, generated, rp=1.0, fp=0.0, pp=0.0):
    """row: bf16 torch tensor [V] (CPU); generated: the token ids generated so far, in any order. Returns a new row."""
    out = row.clone()
    ids, counts = np.unique(np.asarray(list(generated), dtype=np.int64), return_counts=True)
    if is_off(rp, fp, pp) or ids.size == 0:
        return out
    sel = torch.from_numpy(ids)
    l = row[sel].float().numpy()
    rp32, fp32, pp32 = np.float32(rp), np.float32(fp), np.float32(pp)
    with np.errstate(over="ignore", invalid="ignore"):
        # numpy float32 ufuncs round each operation on its own
        r = np.where(l < 0, l * rp32, l / rp32).astype(np.float32)
        r = (r - fp32 * counts.astype(np.float32)).astype(np.float32)
        r = (r - pp32).astype(np.float32)
    new = bits(torch.from_numpy(r).to(torch.bfloat16))        # round to nearest even
    # NaN keeps its bits. Assignments go through int16 views: a bf16 assignment may canonicalise a NaN.
    nan = torch.from_numpy(np.isnan(l))
    out_bits = bits(out)
    out_bits[sel] = torch.where(nan, out_bits[sel], new)
    return out


def bits(t):
    """bf16 tensor -> its int16 bit patterns (NaN-safe equality)."""
    return t.contiguous().view(torch.int16)
