"""bfloat16 storage of dense features, restated in numpy: round to nearest even from f32 (what the device's
__float2bfloat16_rn does) and the exact widening back to f32.  Test infrastructure."""
import numpy as np

CANONICAL_NAN = np.uint16(0x7FC0)


def round_bits(x):
    """f32 array -> the uint16 bits of its bf16 rounding, to nearest, ties to even.  Adding 0x7FFF plus the kept part's lowest
    bit and dropping the low half rounds every finite value and keeps +-Inf (the carry out of the largest finite values lands
    on Inf's bits); a NaN becomes the canonical quiet NaN."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    r[np.isnan(x)] = CANONICAL_NAN
    return r


def widen(bits):
    """uint16 bf16 bits -> f32, exactly: the bits become the f32's upper half"""
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def rounded(x):
    """x rounded to bf16 and widened back: the f32 table a bf16 graph holds"""
    x = np.asarray(x, dtype=np.float32)
    return widen(round_bits(x)).reshape(x.shape)


def special_values():
    """+-0, subnormals, the smallest and largest normals, ties at both parities, values that round up to Inf, +-Inf, and
    quiet and signalling NaNs with payloads"""
    bits = [
        0x00000000, 0x80000000,                          # +-0
        0x00000001, 0x80000001, 0x00007FFF, 0x00008000,  # subnormals: the smallest, below and at a tie
        0x00018000, 0x00028000, 0x007FFFFF, 0x807FFFFF,  # subnormal ties at odd / even kept parity, the largest subnormal
        0x00800000, 0x80800000,                          # smallest normals
        0x7F7FFFFF, 0xFF7FFFFF,                          # largest normals: round up to +-Inf
        0x7F7F7FFF, 0x7F7F8000, 0x7F7F8001, 0x7F7EFFFF,  # around the last tie below Inf
        0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000,  # ties at even and odd kept parity, both signs
        0x3F807FFF, 0x3F808001,                          # just below and above a tie
        0x7F800000, 0xFF800000,                          # +-Inf
        0x7FC00000, 0xFFC00001, 0x7FC12345,              # quiet NaNs with payloads and sign
        0x7F800001, 0xFF80ABCD, 0x7FBFFFFF,              # signalling NaNs with payloads
    ]
    return np.array(bits, dtype=np.uint32).view(np.float32)
