"""Host-side parts of the batched COCO results (no GPU): the one-copy device-to-host helper and the validation of the per-image RLE
canvas sizes, which happens before anything is launched."""
import numpy as np
import pytest
import torch


def test_to_host_splits_one_copy_back_into_typed_arrays():
    from detectorch_b200 import ops
    a = torch.arange(12, dtype=torch.int64).reshape(3, 4)
    b = torch.tensor([1.5, -2.25, 3.0], dtype=torch.float32)
    c = torch.tensor([[7, -8]], dtype=torch.int32)
    d = torch.zeros((0, 5), dtype=torch.float32)
    e = torch.tensor([255, 0, 1], dtype=torch.uint8)
    got = ops.to_host(a, b, c.t(), d, e)                  # a non-contiguous view is copied as its values
    for g, t in zip(got, (a, b, c.t(), d, e)):
        assert g.dtype == t.numpy().dtype and g.shape == tuple(t.shape)
        assert np.array_equal(g, t.numpy())


def test_segm_image_sizes():
    from detectorch_b200 import ops
    sz = ops.segm_image_sizes([(480.9, 640.0), (1, 2)], 2)
    assert sz.dtype == np.int64 and sz.tolist() == [[480, 640], [1, 2]]
    assert ops.segm_image_sizes(torch.tensor([[427, 640]]), 1).tolist() == [[427, 640]]
    assert ops.segm_image_sizes(np.zeros((0, 2)), 0).shape == (0, 2)
    for bad in ([(10, 10)], [(10, 10), (0, 5)], [(10, 10), (5, -3)], [(10, 10), (0.9, 5)], [(10, 10, 1), (5, 5)],
                [(10, 10), (float("nan"), 5)], [(10, 10), (float("inf"), 5)], [(2 ** 16, 2 ** 16), (1, 1)], [10, 10]):
        with pytest.raises(ValueError):
            ops.segm_image_sizes(bad, 2)


def test_batch_results_boxes_per_class_without_masks():
    """Faster R-CNN output (no masks): per image the postprocess_output structures, read from the padded slots up to each count; slots
    that are not class-major are refused."""
    from detectorch_b200.utils import result_utils
    rng = np.random.RandomState(0)
    B, cap, NC = 3, 10, 6
    counts = np.array([7, 0, 10], np.int32)
    boxes = rng.uniform(0, 100, (B, cap, 4)).astype(np.float32)
    scores = rng.uniform(0, 1, (B, cap)).astype(np.float32)
    classes = np.sort(rng.randint(1, NC, (B, cap)), axis=1).astype(np.int32)
    classes[0, 7:] = 0                                                  # dead slots are never read
    out = {"boxes": torch.from_numpy(boxes), "scores": torch.from_numpy(scores), "classes": torch.from_numpy(classes),
           "counts": torch.from_numpy(counts)}
    got = result_utils.batch_results(out, [(200, 300)] * B, num_classes=NC)
    for b in range(B):
        n = counts[b]
        sc, bx, cb, segms = got[b]
        assert segms is None and np.array_equal(sc, scores[b, :n]) and np.array_equal(bx, boxes[b, :n])
        assert len(cb) == NC and cb[0] == []
        for j in range(1, NC):
            m = classes[b, :n] == j
            want = np.hstack((boxes[b, :n][m], scores[b, :n][m][:, None])).astype(np.float32)
            assert cb[j].dtype == np.float32 and cb[j].shape == want.shape and np.array_equal(cb[j], want)
    classes[2, :2] = [3, 1]
    with pytest.raises(RuntimeError):
        result_utils.batch_results(out, [(200, 300)] * B, num_classes=NC)


def test_batch_results_validates_original_sizes_first():
    """Bad original sizes raise ValueError before any device work: here the outputs are CPU tensors, which no kernel could take."""
    from detectorch_b200.utils import result_utils
    out = {"boxes": torch.zeros((2, 100, 4)), "scores": torch.zeros((2, 100)), "classes": torch.zeros((2, 100), dtype=torch.int32),
           "counts": torch.zeros((2,), dtype=torch.int32), "masks": torch.zeros((2, 100, 28, 28))}
    for bad in ([(10, 10)], [(10, 10)] * 3, [(10, 10), (0, 10)], [(10, 10), (10, -1)], [(10, 10, 3)] * 2):
        with pytest.raises(ValueError):
            result_utils.batch_results(out, bad)
