"""numpy restatement of the permutation keys of csrc/importance.cu (dtb_perm_keys)."""
import numpy as np

_M1, _M2 = np.uint64(0xff51afd7ed558ccd), np.uint64(0xc4ceb9fe1a85ec53)
_LOW = np.uint64(0xFFFFFFFF)


def mix32(x):
    """dtb_common.cuh's mix32: the low 32 bits of murmur3's 64-bit finaliser."""
    x = np.asarray(x, np.uint64)
    with np.errstate(over='ignore'):
        x = x ^ (x >> np.uint64(33))
        x = x * _M1
        x = x ^ (x >> np.uint64(33))
        x = x * _M2
        x = x ^ (x >> np.uint64(33))
    return x & _LOW


def perm_keys(seed, iteration, column, rows):
    """int64 keys: ((hash ^ 2^31) << 32) | row."""
    s32 = np.uint64(32)
    a = mix32((np.uint64(seed) << s32) | np.uint64(iteration))
    b = mix32((a << s32) | np.uint64(column))
    r = np.arange(rows, dtype=np.uint64)
    h = mix32((b << s32) | r) ^ np.uint64(0x80000000)
    return ((h << s32) | r).view(np.int64)


def permutation(seed, iteration, column, rows):
    return (np.sort(perm_keys(seed, iteration, column, rows)) & 0xFFFFFFFF).astype(np.int64)
