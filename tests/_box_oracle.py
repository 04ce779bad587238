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


def _contig_strides(shape):
    st, acc = [0] * len(shape), 1
    for d in range(len(shape) - 1, -1, -1):
        st[d] = acc
        acc *= shape[d]
    return st


def _random_strides(rng, sizes):
    """Strides of the box inside a larger, possibly transposed, row-major buffer."""
    nd = len(sizes)
    outer = [max(s, 1) + int(rng.integers(0, 3)) for s in sizes]  # the box is a sub-box of a padded array
    perm = rng.permutation(nd) if rng.random() < 0.4 else np.arange(nd)
    st_perm = _contig_strides([outer[p] for p in perm])
    strides = [0] * nd
    for i, p in enumerate(perm):
        strides[p] = st_perm[i]
    extent = sum((o - 1) * s for o, s in zip(outer, strides)) + 1 if nd else 1
    return strides, extent


def _random_boxes(rng, n_boxes, dst_base):
    """``n_boxes`` random boxes (0-8 dims, element sizes 1-16, padded / transposed strides on both sides) laid out one after
    the other in a source and a destination buffer.  Returns the boxes as ``BoxPlan`` takes them (destinations at
    ``dst_base`` + offset), the same boxes with destination offsets and byte extents, and the source / destination bytes."""
    boxes, cur_src, cur_dst, expect = [], 0, 0, []
    for _ in range(n_boxes):
        nd = int(rng.integers(0, 9))
        sizes = [int(rng.integers(0 if rng.random() < 0.05 else 1, 5)) for _ in range(nd)]
        while np.prod(sizes, dtype=np.int64) > 3000:
            sizes[int(np.argmax(sizes))] -= 1
        elem = int(rng.choice([1, 2, 4, 8, 16]))
        sst, s_ext = _random_strides(rng, sizes)
        dstr, d_ext = _random_strides(rng, sizes)
        src_off = cur_src + int(rng.integers(0, 40))
        dst_off = cur_dst + int(rng.integers(0, 40))
        boxes.append((elem, sizes, src_off, sst, dst_base + dst_off, dstr))
        expect.append((elem, sizes, src_off, sst, dst_off, dstr, s_ext * elem, d_ext * elem))
        cur_src = src_off + s_ext * elem
        cur_dst = dst_off + d_ext * elem
    return boxes, expect, cur_src, cur_dst
