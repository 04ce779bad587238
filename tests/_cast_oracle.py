"""TEST INFRASTRUCTURE: the fp32 / bf16 / fp16 conversions of the converting box scatter restated in numpy, on raw bits.

Narrowing rounds to nearest even, keeps subnormals and sends overflow to +-inf (IEEE, as ``Tensor.to``).  NaN is written
as 0x7FFF by the narrowing conversions; widening keeps whatever NaN comes out, so comparisons treat NaN sign and payload
as unspecified (``nan_aware_equal``)."""
import numpy as np
import torch

CAST_NONE, CAST_F32_BF16, CAST_F32_F16, CAST_BF16_F32, CAST_F16_F32, CAST_BF16_F16, CAST_F16_BF16 = range(7)

# code -> (source dtype, destination dtype)
CAST_DTYPES = {
    CAST_F32_BF16: (torch.float32, torch.bfloat16),
    CAST_F32_F16: (torch.float32, torch.float16),
    CAST_BF16_F32: (torch.bfloat16, torch.float32),
    CAST_F16_F32: (torch.float16, torch.float32),
    CAST_BF16_F16: (torch.bfloat16, torch.float16),
    CAST_F16_BF16: (torch.float16, torch.bfloat16),
}
CAST_OF = {v: k for k, v in CAST_DTYPES.items()}
PAIRS = list(CAST_DTYPES.values())
SIZE = {torch.float32: 4, torch.bfloat16: 2, torch.float16: 2}
UINT = {2: np.uint16, 4: np.uint32}


def _f32_to_bf16(u):
    u = u.astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    r[(u & 0x7FFFFFFF) > 0x7F800000] = 0x7FFF
    return r


def _f32_to_f16(u):
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    with np.errstate(over="ignore", invalid="ignore"):
        r = u.astype(np.uint32).view(np.float32).astype(np.float16).view(np.uint16).copy()
    r[nan] = 0x7FFF
    return r


def _bf16_to_f32(u):
    return u.astype(np.uint32) << 16


def _f16_to_f32(u):
    return u.astype(np.uint16).view(np.float16).astype(np.float32).view(np.uint32)


def convert_bits(code: int, src: np.ndarray) -> np.ndarray:
    """Source element bits (uint16 / uint32 array) -> destination element bits."""
    if code == CAST_F32_BF16:
        return _f32_to_bf16(src)
    if code == CAST_F32_F16:
        return _f32_to_f16(src)
    if code == CAST_BF16_F32:
        return _bf16_to_f32(src)
    if code == CAST_F16_F32:
        return _f16_to_f32(src)
    if code == CAST_BF16_F16:
        return _f32_to_f16(_bf16_to_f32(src))
    if code == CAST_F16_BF16:
        return _f32_to_bf16(_f16_to_f32(src))
    raise ValueError(code)


def convert_bytes(code: int, src: bytes) -> bytes:
    es, ed = SIZE[CAST_DTYPES[code][0]], SIZE[CAST_DTYPES[code][1]]
    return convert_bits(code, np.frombuffer(src, dtype=UINT[es])).astype(UINT[ed]).tobytes()


def nan_mask(bits: np.ndarray, dtype: torch.dtype) -> np.ndarray:
    b = bits.astype(np.uint64)
    if dtype == torch.float32:
        return (b & 0x7FFFFFFF) > 0x7F800000
    if dtype == torch.bfloat16:
        return (b & 0x7FFF) > 0x7F80
    if dtype == torch.float16:
        return (b & 0x7FFF) > 0x7C00
    return np.zeros(b.shape, dtype=bool)


def nan_aware_equal(got: np.ndarray, want: np.ndarray, dtype: torch.dtype) -> bool:
    """Element bits equal, except that where ``want`` is NaN ``got`` only has to be NaN as well."""
    got, want = np.asarray(got).reshape(-1), np.asarray(want).reshape(-1)
    if got.shape != want.shape:
        return False
    wn, gn = nan_mask(want, dtype), nan_mask(got, dtype)
    return bool(np.array_equal(wn, gn) and np.array_equal(got[~wn], want[~wn]))


def tensor_bits(t: torch.Tensor) -> np.ndarray:
    t = t.detach().cpu().contiguous().reshape(-1)
    return t.view({4: torch.int32, 2: torch.int16}[t.element_size()]).numpy().view(UINT[t.element_size()])


def tensors_nan_aware_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype not in SIZE:
        return bytes(a.detach().cpu().contiguous().reshape(-1).view(torch.uint8).numpy()) == bytes(
            b.detach().cpu().contiguous().reshape(-1).view(torch.uint8).numpy())
    return nan_aware_equal(tensor_bits(a), tensor_bits(b), a.dtype)


# fp32 bit patterns at the edges of the conversions
SPECIAL_F32_BITS = np.array(
    [
        0x00000000, 0x80000000,  # +-0
        0x7F800000, 0xFF800000,  # +-inf
        0x7FC00123, 0xFFC00001, 0x7F800001, 0xFFA00000,  # NaNs of both signs, quiet and signalling, with payloads
        0x00000001, 0x807FFFFF, 0x00400000,  # fp32 subnormals (-> bf16 subnormals / 0)
        0x33800000, 0x33C00000, 0x387FC000, 0xB4000000,  # fp16 subnormal results: 2^-24, 1.5 * 2^-24, 2^-15 - ..., -2^-23
        0x33000000, 0x33000001,  # 2^-25: tie to 0 / just above it -> smallest fp16 subnormal
        0x3F808000, 0x3F818000, 0x3F808001,  # bf16 RNE: tie down to even, tie up to even, above the tie
        0x3F801000, 0x3F803000, 0x3F801001,  # fp16 RNE: the same three
        0x477FF000, 0x477FEFFF, 0x477FE000, 0xC77FF000,  # fp16 edge: 65520 -> inf, 65519.99 -> 65504, 65504, -65520 -> -inf
        0x7F7FFFFF, 0xFF7FFFFF,  # fp32 max -> bf16 inf
        0x7F7F7FFF, 0x3F800000, 0xC0490FDB,  # just below the bf16 overflow tie, 1, -pi
    ],
    dtype=np.uint32,
)


def special_tensor(dtype: torch.dtype) -> torch.Tensor:
    """The special values as a tensor of ``dtype`` (fp32 ones converted by torch for the 16-bit formats, plus 16-bit
    NaNs with payloads and 16-bit subnormals written as bits)."""
    f32 = torch.from_numpy(SPECIAL_F32_BITS.view(np.float32).copy())
    if dtype == torch.float32:
        return f32
    extra = np.array([0x7C01, 0xFE00, 0x7FFF, 0xFC01, 0x0001, 0x8001, 0x03FF, 0x0200, 0x7F81, 0xFFC1, 0x007F, 0x8040],
                     dtype=np.uint16)
    x = torch.cat([f32.to(dtype).view(torch.int16), torch.from_numpy(extra.view(np.int16).copy())])
    return x.view(dtype)
