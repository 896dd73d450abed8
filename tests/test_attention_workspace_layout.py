"""CPU: the layout of an attention workspace (include/latex_ocr_b200.h, lo_attention_workspace_bytes).  B int32 ticket counters
sit at offset 0 and the split partials [B][16][C + 2] fp32 after them.  Up to 1,024 rows the partials start at 4096, the layout
of every training, stand-alone and TF-decoder workspace; decoding has no row cap, and above 1,024 rows every row's counter must
still lie in front of the partials, or the ticket of a high row lands in a low row's partial sums."""
import pytest

from latex_ocr_b200 import _lib

MAXSPLIT = 16
RAGGED_CAP = 6144                 # most rows of one decode call (the ragged attention's CTA map)


def _partials(B, C):
    return B * MAXSPLIT * (C + 2) * 4


@pytest.mark.parametrize("C", [256, 512, 1024])
def test_layout_up_to_1024_rows_is_the_fixed_4096_byte_header(C):
    L = _lib.lib()
    for B in (1, 2, 33, 132, 133, 444, 512, 513, 1000, 1023, 1024):
        assert L.lo_attention_workspace_bytes(B, C) == 4096 + _partials(B, C), B
        assert L.lo_decoder_workspace_bytes(B, C) == 2 * (4096 + _partials(B, C)), B


@pytest.mark.parametrize("C", [256, 512, 1024])
def test_every_row_counter_lies_in_front_of_the_partials(C):
    L = _lib.lib()
    prev = 0
    for B in list(range(1, 1300)) + [1536, 2047, 2048, 2049, 4095, 4096, 4097, RAGGED_CAP - 1, RAGGED_CAP]:
        n = L.lo_attention_workspace_bytes(B, C)
        off = n - _partials(B, C)                  # where the partials start
        assert off >= 4 * B and off >= 4096, B
        assert off % 256 == 0, B
        # monotone: a workspace sized for a capacity holds the layout of any smaller launch (the ragged decode cache)
        assert n > prev, B
        prev = n
        assert L.lo_decoder_workspace_bytes(B, C) == 2 * n, B
    # above 1,024 rows the header grows only as far as the counters need (4 bytes a row, rounded up to 256)
    assert L.lo_attention_workspace_bytes(1025, C) - _partials(1025, C) == 4352
    assert L.lo_attention_workspace_bytes(1280, C) - _partials(1280, C) == 5120
