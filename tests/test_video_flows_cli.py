"""`-flow_pattern_forward` of the video CLI: the combinations it refuses (no GPU needed, the refusal comes first)."""
import pytest

from fav_b200 import _lib, video

BASE = ["-input_pattern", "frame_%04d.ppm", "-flow_pattern_forward", "forward_{%d}_[%d].flo"]


def refused(argv):
    with pytest.raises(_lib.FavError) as e:
        video.main(argv)
    return e.value


def test_forward_flows_need_backward_flows():
    e = refused(BASE)
    assert e.status == _lib.FAV_ERR_INVALID and "-flow_pattern" in e.message


def test_computed_certainty_is_not_inverted():
    e = refused(BASE + ["-flow_pattern", "backward_[%d]_{%d}.flo", "-invert_occlusion"])
    assert e.status == _lib.FAV_ERR_INVALID and "-invert_occlusion" in e.message


def test_certainty_pgms_or_forward_flows():
    e = refused(BASE + ["-flow_pattern", "backward_[%d]_{%d}.flo", "-occlusions_pattern", "reliable_[%d]_{%d}.pgm"])
    assert e.status == _lib.FAV_ERR_INVALID
