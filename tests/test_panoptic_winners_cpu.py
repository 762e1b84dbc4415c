"""CPU: ape_panoptic_winners validates its arguments before any CUDA call (so this runs without a device), and the segment
bookkeeping that the device path shares with postprocess_panoptic decides segments from the three areas as the reference does."""
import torch

from ape_b200.modeling.postprocess import _segments


def test_arguments_are_rejected_before_any_cuda_call(built):
    import ape_b200

    lib = ape_b200._lib.lib
    F16 = ape_b200._lib.APE_DTYPE_F16
    geo = (16, 16, 32, 32, 30, 20, 8, 8)  # logits, padded, image, output
    assert lib.ape_panoptic_winners(None, None, None, None, None, 3, *geo, 0.5, 7, None) == -1
    assert b"dtype" in lib.ape_last_error()
    assert lib.ape_panoptic_winners(None, None, None, None, None, 4097, *geo, 0.5, F16, None) == -1
    assert b"4096" in lib.ape_last_error()
    assert lib.ape_panoptic_winners(None, None, None, None, None, 3, 16, 16, 32, 32, 33, 20, 8, 8, 0.5, F16, None) == -1
    assert lib.ape_panoptic_winners(None, None, None, None, None, 3, 16, 16, 32, 32, 30, 20, 0, 8, 0.5, F16, None) == -1
    assert lib.ape_panoptic_winners(None, None, None, None, None, 3, *geo, 0.5, F16, None) == -3


def test_segments_bookkeeping():
    # columns: mask_area, original_area, inter_area, class; things are classes 0 and 1
    stats = torch.tensor([[50, 40, 0, 30, 30, 5, 10],
                          [60, 200, 9, 40, 50, 5, 12],
                          [45, 30, 0, 25, 20, 5, 9],
                          [0, 1, 1, 5, 5, 1, 7]])
    lut, info = _segments(stats, [0, 1], 2, True, 0.4)
    # k=0 thing; k=1 area / orig = 0.2 < 0.4 dropped; k=2 no pixel; k=3 stuff 5 -> new segment; k=4 stuff 5 again -> merged;
    # k=5 thing 1; k=6 stuff 7
    assert lut.tolist() == [1, 0, 0, 2, 2, 3, 4]
    assert info == [{"id": 1, "isthing": True, "category_id": 0}, {"id": 2, "isthing": False, "category_id": 4},
                    {"id": 3, "isthing": True, "category_id": 1}, {"id": 4, "isthing": False, "category_id": 6}]
