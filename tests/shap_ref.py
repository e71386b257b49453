"""float64 restatement of Kernel SHAP as shap's KernelExplainer runs it (identity link, no L1 selection), written as
shap's loops, for deeptables_b200/explain.py.  The random coalitions consume the generator as the product does: the
sizes by one ``choice`` call, then M uniform keys per draw, the mask being the columns of the ``size`` smallest."""
import itertools
from math import comb

import numpy as np


def budget(M, nsamples):
    n = 2 * M + 2 ** 11 if nsamples == 'auto' else nsamples
    if M <= 30 and n > 2 ** M - 2:
        n = 2 ** M - 2
    return n


def not_equal(i, j):
    if isinstance(i, (int, float, np.number)) and isinstance(j, (int, float, np.number)):
        return 0 if np.isclose(i, j, equal_nan=True) else 1
    return 0 if i == j else 1


def varying(x, data):
    """x: [columns] values, data: [rows, columns] object array."""
    out = []
    for i in range(data.shape[1]):
        if np.sum(np.frompyfunc(not_equal, 2, 1)(x[i], data[:, i])) > 0:
            out.append(i)
    return out


def coalitions(M, nsamples, rng):
    """shap's explain(): the enumerated sizes, then the drawn masks.  -> (masks [K, M] float64, weights [K])."""
    n = budget(M, nsamples)
    num_subset_sizes = int(np.ceil((M - 1) / 2.0))
    num_paired_subset_sizes = int(np.floor((M - 1) / 2.0))
    weight_vector = np.array([(M - 1.0) / (i * (M - i)) for i in range(1, num_subset_sizes + 1)])
    weight_vector[:num_paired_subset_sizes] *= 2
    weight_vector /= np.sum(weight_vector)
    masks, weights = [], []

    def add(mask, w):
        masks.append(mask.copy())
        weights.append(w)

    num_full_subsets = 0
    num_samples_left = n
    mask = np.zeros(M)
    remaining_weight_vector = weight_vector.copy()
    for subset_size in range(1, num_subset_sizes + 1):
        nsubsets = comb(M, subset_size)
        if subset_size <= num_paired_subset_sizes:
            nsubsets *= 2
        if num_samples_left * remaining_weight_vector[subset_size - 1] / nsubsets >= 1.0 - 1e-8:
            num_full_subsets += 1
            num_samples_left -= nsubsets
            if remaining_weight_vector[subset_size - 1] < 1.0:
                remaining_weight_vector /= (1 - remaining_weight_vector[subset_size - 1])
            w = weight_vector[subset_size - 1] / comb(M, subset_size)
            if subset_size <= num_paired_subset_sizes:
                w /= 2.0
            for inds in itertools.combinations(range(M), subset_size):
                mask[:] = 0.0
                mask[np.array(inds, dtype='int64')] = 1.0
                add(mask, w)
                if subset_size <= num_paired_subset_sizes:
                    mask[:] = np.abs(mask - 1)
                    add(mask, w)
        else:
            break

    nfixed_samples = len(masks)
    samples_left = n - nfixed_samples
    if num_full_subsets != num_subset_sizes and samples_left > 0:
        remaining_weight_vector = weight_vector.copy()
        remaining_weight_vector[:num_paired_subset_sizes] /= 2
        remaining_weight_vector = remaining_weight_vector[num_full_subsets:]
        remaining_weight_vector /= np.sum(remaining_weight_vector)
        ind_set = rng.choice(len(remaining_weight_vector), 4 * samples_left, p=remaining_weight_vector)
        ind_set_pos = 0
        used_masks = {}
        while samples_left > 0 and ind_set_pos < len(ind_set):
            mask.fill(0.0)
            ind = ind_set[ind_set_pos]
            ind_set_pos += 1
            subset_size = ind + num_full_subsets + 1
            mask[np.argsort(rng.random_sample(M))[:subset_size]] = 1.0
            mask_tuple = tuple(mask)
            new_sample = False
            if mask_tuple not in used_masks:
                new_sample = True
                used_masks[mask_tuple] = len(masks)
                samples_left -= 1
                add(mask, 1.0)
            else:
                weights[used_masks[mask_tuple]] += 1.0
            if samples_left > 0 and subset_size <= num_paired_subset_sizes:
                mask[:] = np.abs(mask - 1)
                if new_sample:
                    samples_left -= 1
                    add(mask, 1.0)
                else:
                    weights[used_masks[mask_tuple] + 1] += 1.0
        weight_left = np.sum(weight_vector[num_full_subsets:])
        w = np.array(weights[nfixed_samples:])
        weights[nfixed_samples:] = list(w * (weight_left / w.sum()))
    return np.array(masks), np.array(weights)


def solve(masks, weights, ey, fx, fnull):
    """shap's solve(): eliminate the last column under sum(phi) = f(x) - E, then inv(Z'WZ) Z'Wy."""
    eyAdj = ey - fnull
    eyAdj2 = eyAdj - masks[:, -1] * (fx - fnull)
    etmp = np.transpose(np.transpose(masks[:, :-1]) - masks[:, -1])
    tmp = np.transpose(np.transpose(etmp) * np.transpose(weights))
    w = np.dot(np.linalg.inv(np.dot(np.transpose(tmp), etmp)), np.dot(np.transpose(tmp), eyAdj2))
    phi = np.zeros(masks.shape[1])
    phi[:-1] = w
    phi[-1] = (fx - fnull) - sum(w)
    return phi


def exact_shapley(value, M):
    """phi_i = sum over S not holding i of |S|! (M-|S|-1)! / M! (v(S + i) - v(S)); ``value(frozenset)`` -> float."""
    from math import factorial
    v = {S: value(frozenset(S)) for r in range(M + 1) for S in itertools.combinations(range(M), r)}
    phi = np.zeros(M)
    for i in range(M):
        for S, vs in v.items():
            if i in S:
                continue
            w = factorial(len(S)) * factorial(M - len(S) - 1) / factorial(M)
            phi[i] += w * (v[tuple(sorted(S + (i,)))] - vs)
    return phi
