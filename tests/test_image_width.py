"""The scan-image rule (sdx_image_width, host only): which byte-aligned width a column of one batch gets, at its edges."""
import pytest

from snappydata_b200 import capi

INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1
LONG_MIN, LONG_MAX = -2 ** 63, 2 ** 63 - 1


@pytest.fixture(scope="module")
def api():
    return capi.product_api()


@pytest.mark.parametrize("elem_bytes", [4, 8])
def test_dictionary_images_hold_at_most_256_bit_patterns(api, elem_bytes):
    assert capi.image_width(api, True, elem_bytes, ndistinct=1) == 1
    assert capi.image_width(api, True, elem_bytes, ndistinct=256) == 1
    assert capi.image_width(api, True, elem_bytes, ndistinct=257) == 0


@pytest.mark.parametrize("elem_bytes,span,want", [
    (4, 255, 1), (4, 256, 2), (4, 65535, 2), (4, 65536, 0),
    (2, 255, 1), (2, 256, 0),
    (8, 255, 1), (8, 256, 2), (8, 65535, 2), (8, 65536, 0)])
def test_frame_of_reference_width_follows_the_range(api, elem_bytes, span, want):
    for lo in (0, -7, -span):
        assert capi.image_width(api, False, elem_bytes, lo=lo, hi=lo + span) == want, (elem_bytes, span, lo)


def test_full_integer_spans_keep_the_verbatim_bytes(api):
    assert capi.image_width(api, False, 4, lo=INT_MIN, hi=INT_MAX) == 0
    assert capi.image_width(api, False, 8, lo=INT_MIN, hi=INT_MAX) == 0
    assert capi.image_width(api, False, 8, lo=LONG_MIN, hi=LONG_MAX) == 0
    assert capi.image_width(api, False, 8, lo=LONG_MAX - 255, hi=LONG_MAX) == 1
    assert capi.image_width(api, False, 8, lo=LONG_MIN, hi=LONG_MIN + 65535) == 2


def test_bad_element_width_is_refused(api):
    with pytest.raises(capi.SdError):
        capi.image_width(api, False, 3, lo=0, hi=1)
