"""TEST INFRASTRUCTURE: the box scatter restated in numpy -- what torch's ``FileSystemReader.read_data`` does per read item
(``narrow_tensor_by_index`` of the saved chunk, then ``target.copy_()``), on raw byte buffers."""
import numpy as np


def box_copy(src: np.ndarray, dst: np.ndarray, elem: int, sizes, src_off: int, src_strides, dst_off: int, dst_strides) -> None:
    """Element (i_0, ..., i_k) of the box -- ``elem`` bytes at byte ``src_off + sum i_d * src_strides[d] * elem`` of the uint8
    buffer ``src`` -- goes to byte ``dst_off + sum i_d * dst_strides[d] * elem`` of ``dst``."""
    sizes = [int(s) for s in sizes]
    if any(s == 0 for s in sizes):
        return

    def index(off, strides):
        idx = np.full(sizes, off, dtype=np.int64)
        for d, (n, st) in enumerate(zip(sizes, strides)):
            shape = [1] * len(sizes)
            shape[d] = n
            idx = idx + (np.arange(n, dtype=np.int64) * st * elem).reshape(shape)
        return idx.reshape(-1, 1) + np.arange(elem, dtype=np.int64)

    dst[index(dst_off, dst_strides)] = src[index(src_off, src_strides)]
