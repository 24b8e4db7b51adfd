"""Host-side mirror of Jlama's tensor types (core/tensor/*): the operands the TensorOperations
plug-in receives.  Storage is numpy (the stand-in for Java's off-heap MemorySegments); the block
formats and quantiser arithmetic follow the reference bit for bit:

  FloatBufferTensor      core/tensor/FloatBufferTensor.java
  BFloat16BufferTensor   core/tensor/BFloat16BufferTensor.java + core/math/FloatConversions.java:31-90
  Q8ByteBufferTensor     core/tensor/Q8ByteBufferTensor.java:37-223   (int8 + f32 scale per 32)
  Q4ByteBufferTensor     core/tensor/Q4ByteBufferTensor.java:34-259   (byte j = q[j] | q[j+16] << 4)
"""
import uuid

import numpy as np

from .native import BF16, F32, I8, Q4

BLOCK = 32
_MIN_VALUE = np.float32(1.401298464324817e-45)  # Float.MIN_VALUE


def float32_to_bfloat16(x):
    """FloatConversions.float32ToBFloat16 (:35-61): round-to-nearest-even, NaN preserving."""
    bits = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    s = (bits >> 16) & 0x8000
    e = (bits >> 16) & 0x7F80
    m = bits & 0x7FFFFF
    mshift = m >> 16
    masked = (m & 0xFFFF).astype(np.int64)
    cmp = masked - 0x8000
    m1 = np.where(cmp > 0, mshift + 1, np.where(cmp < 0, mshift, np.where(mshift & 1, mshift + 1, mshift)))
    normal = (s | (e + m1)).astype(np.uint16)
    sentinel = np.where(m != 0, np.uint16(0x7FC0), (bits >> 16).astype(np.uint16))
    return np.where(e != 0x7F80, normal, sentinel).astype(np.uint16)


def bfloat16_to_float32(raw):
    """FloatConversions.bFloat16ToFloat32 (:31-33)."""
    return (np.ascontiguousarray(raw, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def quantize_q4(x):
    """Q4ByteBufferTensor(AbstractTensor) (:45-120): returns (packed uint8 [rows, cols/2], scales [rows, cols/32])."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    rows, cols = x.shape
    assert cols % BLOCK == 0
    b = x.reshape(rows, cols // BLOCK, BLOCK)
    ab = np.abs(b)
    idx = np.argmax(ab, axis=2)  # first index of the largest |v| (strict '>' scan :74-81)
    mx = np.take_along_axis(b, idx[..., None], axis=2)[..., 0]
    amax = np.take_along_axis(ab, idx[..., None], axis=2)[..., 0]
    mx = np.where(amax > _MIN_VALUE, mx, _MIN_VALUE).astype(np.float32)
    with np.errstate(divide="ignore", over="ignore", invalid="ignore", under="ignore"):
        scale = (mx / np.float32(-8.0)).astype(np.float32)
        iscale = np.where(scale != 0, np.float32(1.0) / scale, np.float32(0.0)).astype(np.float32)
        f = (b * iscale[..., None]).astype(np.float32) + np.float32(8.5)
        f = np.where(np.isnan(f), np.float32(0), f)
        # (int) saturates: clipped in double, where 2^31 - 1 is exact (in float it rounds to 2^31, which would wrap to 0, not -1)
        qi = np.clip(np.trunc(f.astype(np.float64)), -2147483648.0, 2147483647.0).astype(np.int64)
    qi = ((qi + 128) % 256 - 128)  # (byte) wraps
    qi = np.minimum(qi, 15)
    lo = qi[..., :16] & 0xFF
    hi = qi[..., 16:]
    packed = (lo | (hi << 4)) & 0xFF
    return packed.astype(np.uint8).reshape(rows, cols // 2), scale


def dequantize_q4(q, scales):
    """Q4ByteBufferTensor.get (:179-197)."""
    rows, half = q.shape
    b = q.reshape(rows, half // 16, 16)
    lo = (b & 0x0F).astype(np.int32) - 8
    hi = ((b >> 4) & 0x0F).astype(np.int32) - 8
    v = np.concatenate([lo, hi], axis=2).astype(np.float32) * scales[..., None].astype(np.float32)
    return v.reshape(rows, half * 2)


def quantize_q8_weights(x):
    """Q8ByteBufferTensor(AbstractTensor) (:45-90): q = (byte)Math.round(x * (127f/max))."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    rows, cols = x.shape
    b = x.reshape(rows, cols // BLOCK, BLOCK)
    mx = np.maximum(np.abs(b).max(axis=2), _MIN_VALUE).astype(np.float32)
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        iscale = (np.float32(127.0) / mx).astype(np.float32)
        scale = np.where(iscale != 0, np.float32(1.0) / iscale, np.float32(0.0)).astype(np.float32)
        f = (b * iscale[..., None]).astype(np.float32)
        r = np.floor(f.astype(np.float64) + 0.5)  # Math.round(float)
        r = np.where(np.isnan(r), 0.0, r)
    qi = np.clip(r, -2147483648.0, 2147483647.0).astype(np.int64)
    qi = (qi + 128) % 256 - 128
    return qi.astype(np.int8).reshape(rows, cols), scale


def quantize_q8_activations(x, offset=0, length=None):
    """TensorOperations.quantize(t, I8, ..) as the Panama back-end does it
    (PanamaTensorOperations.java:1684-1723): d = max/127, q = (byte)(x*(127/max) + 0.5f) truncating."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    rows, cols = x.shape
    length = cols - offset if length is None else length
    q = np.zeros((rows, cols), dtype=np.int8)
    s = np.zeros((rows, cols // BLOCK), dtype=np.float32)
    b = x[:, offset:offset + length].reshape(rows, length // BLOCK, BLOCK)
    mx = np.abs(b).max(axis=2).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        d = (mx / np.float32(127.0)).astype(np.float32)
        idv = np.where(mx != 0, np.float32(127.0) / mx, np.float32(0.0)).astype(np.float32)
        f = ((b * idv[..., None]).astype(np.float32) + np.float32(0.5)).astype(np.float32)
    # F2B narrows through int: NaN -> 0, (int) saturates (an infinite x * id, from a block of subnormals, becomes -1 or 0)
    qi = np.where(np.isnan(f), 0.0, np.clip(np.trunc(f.astype(np.float64)), -2147483648.0, 2147483647.0)).astype(np.int64)
    qi = (qi + 128) % 256 - 128
    q[:, offset:offset + length] = qi.reshape(rows, length).astype(np.int8)
    s[:, offset // BLOCK:(offset + length) // BLOCK] = d
    return q, s


class AbstractTensor:
    """core/tensor/AbstractTensor.java:45-323 (the parts the operator API touches)."""
    dtype = None

    def __init__(self, data, scales=None):
        self.data = np.ascontiguousarray(data)
        self.scales = None if scales is None else np.ascontiguousarray(scales, dtype=np.float32)
        self.uid = uuid.uuid4().hex  # AbstractTensor.getUid() :57,73-79

    @property
    def rows(self):
        return self.data.shape[0]

    @property
    def cols(self):
        return self.data.shape[1]

    def shape(self):
        return (self.rows, self.cols)

    # ---- sparse shapes (core/tensor/TensorShape.java:37-44,94-133): a tensor may STORE only a column range
    # [sparse_col_off, sparse_col_off + cols) or a row range [sparse_row_off, sparse_row_off + rows) of its logical
    # shape; callers keep using logical indices and every operator rebases them (NativeSimdTensorOperations.java:96-107)
    sparse_col_off = 0
    sparse_row_off = 0
    logical_shape = None

    def is_sparse(self):
        return self.logical_shape is not None

    def get_offset(self, row, col):
        """TensorShape.getOffset(row, col) (:94-99): element offset inside the stored buffer."""
        return self.cols * (row - self.sparse_row_off) + col - self.sparse_col_off

    def _column_slice(self, offset, length):
        raise NotImplementedError

    def sparsify(self, offset, length):
        """AbstractTensor.sparsify (core/tensor/AbstractTensor.java:151-172): copy of the column range, logical indices kept."""
        if self.is_sparse() or length == self.cols:
            return self
        t = self._column_slice(offset, length)
        t.sparse_col_off, t.logical_shape = offset, (self.rows, self.cols)
        return t

    def sparsify_rows(self, offset, length):
        """TensorShape.sparseRow (:41-44): the row-range counterpart (jlama-net's row split of a weight)."""
        if self.is_sparse() or length == self.rows:
            return self
        t = self._row_slice(offset, length)
        t.sparse_row_off, t.logical_shape = offset, (self.rows, self.cols)
        return t

    def _row_slice(self, offset, length):
        t = self._column_slice(0, self.cols)
        t.data = np.ascontiguousarray(t.data[offset:offset + length])
        if t.scales is not None:
            t.scales = np.ascontiguousarray(t.scales[offset:offset + length])
        return t

    def get(self, row, col):
        """AbstractTensor.get with logical indices; outside the stored range it raises (TestParser.testSparsify)."""
        r, c = row - self.sparse_row_off, col - self.sparse_col_off
        if not (0 <= r < self.rows and 0 <= c < self.cols):
            raise IndexError("(%d, %d) is outside the stored range of this sparse tensor" % (row, col))
        return float(self.to_float()[r, c])

    def to_float(self):
        raise NotImplementedError

    def quantize(self, dtype):
        """AbstractTensor.quantize (:282-298): never widens, 1-row tensors keep their dtype."""
        if self.dtype == dtype or self.rows == 1 or self.dtype in (Q4, I8):
            return self
        f = self.to_float()
        if dtype == Q4:
            return Q4ByteBufferTensor.from_float(f)
        if dtype == I8:
            return Q8ByteBufferTensor.from_float(f)
        if dtype == BF16:
            return BFloat16BufferTensor.from_float(f)
        if dtype == F32:
            return FloatBufferTensor(f)
        raise ValueError(dtype)


class FloatBufferTensor(AbstractTensor):
    dtype = F32

    def __init__(self, data):
        super().__init__(np.asarray(data, dtype=np.float32))

    def to_float(self):
        return self.data

    def _column_slice(self, offset, length):
        return FloatBufferTensor(self.data[:, offset:offset + length].copy())


class BFloat16BufferTensor(AbstractTensor):
    dtype = BF16

    @classmethod
    def from_float(cls, x):
        return cls(float32_to_bfloat16(x))

    def __init__(self, raw):
        super().__init__(np.asarray(raw, dtype=np.uint16))

    def to_float(self):
        return bfloat16_to_float32(self.data)

    def _column_slice(self, offset, length):
        return BFloat16BufferTensor(self.data[:, offset:offset + length].copy())


class Q8ByteBufferTensor(AbstractTensor):
    dtype = I8

    @classmethod
    def from_float(cls, x):
        return cls(*quantize_q8_weights(x))

    def __init__(self, q, scales):
        super().__init__(np.asarray(q, dtype=np.int8), scales)

    def to_float(self):
        return (self.data.astype(np.float32).reshape(self.rows, -1, BLOCK) * self.scales[..., None]).reshape(self.rows, -1)

    def _column_slice(self, offset, length):
        assert offset % BLOCK == 0 and length % BLOCK == 0
        return Q8ByteBufferTensor(self.data[:, offset:offset + length].copy(), self.scales[:, offset // BLOCK:(offset + length) // BLOCK].copy())


class Q4ByteBufferTensor(AbstractTensor):
    dtype = Q4

    @classmethod
    def from_float(cls, x):
        return cls(*quantize_q4(x))

    def __init__(self, packed, scales):
        super().__init__(np.asarray(packed, dtype=np.uint8), scales)

    @property
    def cols(self):
        return self.data.shape[1] * 2

    def to_float(self):
        return dequantize_q4(self.data, self.scales)

    def _column_slice(self, offset, length):
        assert offset % BLOCK == 0 and length % BLOCK == 0
        return Q4ByteBufferTensor(self.data[:, offset // 2:(offset + length) // 2].copy(), self.scales[:, offset // BLOCK:(offset + length) // BLOCK].copy())
