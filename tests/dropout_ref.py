"""numpy statement of the dropout masks of the kernels (dtb_common.cuh mix32 / dropout_key, dense_bn_loss.cu
dropout_kernel, pnn_attention.cu attention kernels): element i of a call with seed s is kept when
mix32(s * 0x9E3779B97F4A7C15 + i) >= rate * 2^32, all in 64-bit wrap-around arithmetic."""
import numpy as np

GOLDEN = np.uint64(0x9E3779B97F4A7C15)
SEED_MASK = 0xFFFFFFFFFFFF


def mix32(x):
    x = np.asarray(x, dtype=np.uint64).copy()
    with np.errstate(over='ignore'):
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xff51afd7ed558ccd)
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xc4ceb9fe1a85ec53)
        x ^= x >> np.uint64(33)
    return (x & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def threshold(rate):
    """the kernels receive the rate as a float"""
    return np.uint32(int(float(np.float32(rate)) * 4294967296.0))


def bits(seed, index):
    with np.errstate(over='ignore'):
        return mix32(np.uint64(seed) * GOLDEN + np.asarray(index, dtype=np.uint64))


def keep(seed, index, rate):
    return bits(seed, index) >= threshold(rate)


def scale(rate):
    return np.float32(1.0) / (np.float32(1.0) - np.float32(rate))


def attention_keep(seed, rate, rows, heads, fields, row_offset=0):
    """[rows, heads, fields (query), fields (key)] mask of the attention weights: element index
    ((b * heads + h) * F + q) * F + k, b counted from row_offset"""
    n = rows * heads * fields * fields
    index = np.arange(n, dtype=np.uint64) + np.uint64(row_offset * heads * fields * fields)
    return keep(seed, index, rate).reshape(rows, heads, fields, fields)
