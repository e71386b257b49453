"""numpy restatement of expected gradients (deeptables_b200/explain.py gradient_values, csrc/gradshap.cu): the draws,
the interpolated inputs, the per-pair column values and the per-row means, with the kernels' rounding and order."""
import numpy as np


def draws(seed, i, nsamples, bg_rows):
    """Background rows, then alphas (multiples of 2^-24 below 1), from RandomState([seed, i])."""
    rng = np.random.RandomState([seed, i])
    j = rng.randint(0, bg_rows, size=nsamples).astype(np.int32)
    alpha = (np.floor(rng.random_sample(nsamples) * 2.0 ** 24) / 2.0 ** 24).astype(np.float32)
    return j, alpha


def rows_of(table, row_offsets, ids, dims):
    """[P, F, Dmax] float32 embedding rows of ids [P, F] (an id out of range reads as zeros; coordinates past a field's
    width are zero)."""
    P, F = ids.shape
    out = np.zeros((P, F, table.shape[1]), np.float32)
    for f in range(F):
        v = row_offsets[f + 1] - row_offsets[f]
        ok = (ids[:, f] >= 0) & (ids[:, f] < v)
        out[ok, f, :dims[f]] = table[row_offsets[f] + ids[ok, f], :dims[f]]
    return out


def compose(x_cat, x_cont, bg_cat, bg_cont, table, row_offsets, dims, x_index, bg_index, alpha):
    """(emb [P, F, Dmax] (zero past each width), cont [P, C]): b + alpha * (x - b), each operation rounded in float32."""
    a = alpha.astype(np.float32)
    emb = None
    if x_cat is not None and x_cat.shape[1]:
        ei = rows_of(table, row_offsets, x_cat[x_index], dims)
        ej = rows_of(table, row_offsets, bg_cat[bg_index], dims)
        emb = ej + a[:, None, None] * (ei - ej)          # numpy float32: one rounding per operation
    cont = None
    if x_cont is not None and x_cont.shape[1]:
        xv, bv = x_cont[x_index], bg_cont[bg_index]
        cont = bv + a[:, None] * (xv - bv)
    return emb, cont


def reduce(x_cat, x_cont, bg_cat, bg_cont, table, row_offsets, dims, x_index, bg_index, g_emb, g_cont):
    """[P, F + C] float64: per field sum over d in order of g * (E_x - E_b) (float32 difference, float64 product and
    sum; a zero difference skipped), per continuous column g * (x - b).  g_emb: [P, F, Dmax]."""
    parts = []
    if x_cat is not None and x_cat.shape[1]:
        ei = rows_of(table, row_offsets, x_cat[x_index], dims)
        ej = rows_of(table, row_offsets, bg_cat[bg_index], dims)
        delta = (ei - ej).astype(np.float64)
        with np.errstate(invalid='ignore'):
            prod = np.where(delta != 0, g_emb.astype(np.float64) * delta, 0.0)
        acc = np.zeros(prod.shape[:2])
        for d in range(prod.shape[2]):
            acc = acc + prod[:, :, d]
        parts.append(acc)
    if x_cont is not None and x_cont.shape[1]:
        delta = (x_cont[x_index] - bg_cont[bg_index]).astype(np.float64)
        with np.errstate(invalid='ignore'):
            parts.append(np.where(delta != 0, g_cont.astype(np.float64) * delta, 0.0))
    return np.concatenate(parts, axis=1)


def means(values, rows, nsamples):
    """[rows, cols]: each row's samples added in order, then divided by nsamples."""
    v = values.reshape(rows, nsamples, -1)
    acc = np.zeros((rows, v.shape[2]))
    for s in range(nsamples):
        acc = acc + v[:, s]
    return acc / nsamples
