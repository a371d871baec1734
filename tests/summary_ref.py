"""Test infrastructure: a numpy stand-in for the two device reductions behind bayes_js_b200.summary.CudaBlockReducer
(amwg_summary_moments / amwg_summary_digit_hist), so that the host logic and the collectives run on CPU tensors.
Never imported by the product."""
import numpy as np


class NumpyBlockReducer:
    def moments(self, block):
        x = block.numpy()                                    # [rows, entries, chains]
        rows, entries, chains = x.shape
        m = x.sum(axis=0) / rows                             # [entries, chains]
        m2 = ((x - m[None]) ** 2).sum(axis=0)
        out = np.empty((entries, 4))
        for e in range(entries):
            mean = m[e].mean()
            out[e] = (chains, mean, ((m[e] - mean) ** 2).sum(), m2[e].sum())
        return out

    def digit_counts(self, block, npass, prefix_table):
        import torch
        from bayes_js_b200.summary import double_to_key
        x = block.numpy()
        rows, entries, chains = x.shape
        n_prefix = prefix_table.shape[1]
        counts = np.zeros((entries, n_prefix, 256), dtype=np.int64)
        shift = np.uint64(56 - 8 * npass)
        for e in range(entries):
            k = double_to_key(x[:, e, :].ravel())
            digit = ((k >> shift) & np.uint64(255)).astype(np.int64)
            hi = (k >> (shift + np.uint64(8))) if npass else np.zeros_like(k)
            for q in range(n_prefix):
                sel = digit if npass == 0 else digit[hi == prefix_table[e, q]]
                counts[e, q] = np.bincount(sel, minlength=256)
        return torch.from_numpy(counts)


class ChanBlockReducer(NumpyBlockReducer):
    """NumpyBlockReducer whose moments merge per-chain records (1, chain mean, 0, within-chain M2) in a fixed binary tree with
    the Chan merge of the device (merge_moment_records), as amwg_summary_moments' CTA tree does: a chain whose mean is +inf
    merged with a finite one gives the mean NaN there too, where numpy.mean gives +inf."""

    def moments(self, block):
        from bayes_js_b200.summary import merge_moment_records
        x = block.numpy()
        rows, entries, chains = x.shape
        m = x.sum(axis=0) / rows
        with np.errstate(invalid="ignore"):
            m2 = ((x - m[None]) ** 2).sum(axis=0)
        w = 1
        while w < chains:
            w *= 2
        rec = np.zeros((w, entries, 4))
        rec[:chains, :, 0] = 1.0
        rec[:chains, :, 1] = m.T
        rec[:chains, :, 3] = m2.T
        while w > 1:                                         # sh[t] = merge(sh[t], sh[t + w]) for t < w, w halving
            w //= 2
            rec[:w] = merge_moment_records([rec[:w].reshape(-1, 4), rec[w:2 * w].reshape(-1, 4)]).reshape(w, entries, 4)
        return rec[0]


def numpy_summary(x, probs):
    """x [rows, entries, chains] -> (mean, sd, rhat, quantiles) straight from numpy, as a user of sample() would compute them."""
    rows, entries, chains = x.shape
    flat = np.moveaxis(x, 1, 0).reshape(entries, -1)
    mean = flat.mean(axis=1)
    sd = flat.std(axis=1, ddof=1)
    W = x.var(axis=0, ddof=1).mean(axis=1) if rows > 1 else np.full(entries, np.nan)
    B_over_n = x.mean(axis=0).var(axis=1, ddof=1) if chains > 1 else np.full(entries, np.nan)
    with np.errstate(invalid="ignore", divide="ignore"):
        rhat = np.sqrt(((rows - 1) / rows * W + B_over_n) / W)
    q = np.quantile(flat, probs, axis=1) if len(probs) else np.empty((0, entries))
    return mean, sd, rhat, q
