"""CPU: the host model of the block-parallel entropy decode (tests/jpeg_sync_model.py) against tests/jpeg_oracle.py on
every fixture of tests/jpeg_fixtures.py: the converged entry of every subsequence is the true decode's state at its
first bit, and the counts and DC sums the write pass starts from give exactly the oracle's coefficients.  Also the
bounds the kernel relies on: the subsequence count never exceeds the CTA's threads, and the restart-segment table fits
the plane region it borrows."""
import functools

import numpy as np
import pytest

import jpeg_oracle as JO
import jpeg_sync_model as M
from jpeg_fixtures import encode, fixtures, make_image

SEG_BYTES = 20  # struct JSeg (csrc/jpeg.cu)


@functools.lru_cache(maxsize=None)
def model_run():
    """per fixture: (label, rounds, converged == serial, coefficients == oracle, error flag, nsub, nseg, blocks)"""
    out = []
    for label, data in fixtures():
        r = M.decode(data)
        im = r["image"]
        ref = JO.entropy_decode(im.b, im.d, im.g)
        same_coef = all(np.array_equal(a, b) for a, b in zip(r["coef"], ref))
        serial = M.serial_states(im)
        synced = serial == r["exits"][:-1] and serial == r["entries"][1:]
        out.append((label, r["rounds"], synced, same_coef, r["err"], r["nsub"], im.needed, im.total))
    return out


def test_converged_entries_are_the_true_states():
    wrong = [row[0] for row in model_run() if not row[2]]
    assert not wrong, wrong[:20]


def test_counts_and_dc_sums_give_the_oracles_coefficients():
    wrong = [row[0] for row in model_run() if not row[3] or row[4]]
    assert not wrong, wrong[:20]


def test_some_fixture_needs_three_or_more_rounds():
    rounds = sorted(((row[1], row[0]) for row in model_run()), reverse=True)
    print(f"most sync rounds over {len(rounds)} fixtures: {rounds[0][0]} ({rounds[0][1]}); "
          f"fixtures with >= 3 rounds: {sum(r >= 3 for r, _ in rounds)}")
    assert rounds[0][0] >= 3


def test_segment_table_and_records_fit():
    for label, _, _, _, _, nsub, needed, blocks in model_run():
        assert 1 <= nsub <= M.T, label
        assert needed * SEG_BYTES <= blocks * 64, label
    # the worst case: a restart interval of one MCU of one block (grayscale), one segment per block
    assert SEG_BYTES <= 64


@pytest.mark.parametrize("ncomp,per_mcu", [(1, 1), (3, 3), (3, 6), (3, 10)])
def test_subsequence_count_stays_within_the_cta(ncomp, per_mcu):
    """Up to 65535 x 65535 pixels at the most bits a block can take (a 16-bit DC code + 15 bits, then 63 coefficients
    of a 16-bit code + 15 bits each), capped at the 4 GiB a scan can have."""
    worst_block = 16 + 15 + 63 * (16 + 15)
    mcus = (65535 // 8 + 1) ** 2
    top = min(mcus * per_mcu * worst_block, 8 * (1 << 32))
    for bits in [0, 1, 2047, 2048, 2049, M.T * M.S_MIN - 1, M.T * M.S_MIN, M.T * M.S_MIN + 1, 10 ** 9, top - 1, top]:
        S, nsub = M.sub_bits(bits)
        assert S % 32 == 0 and S >= M.S_MIN and 1 <= nsub <= M.T and nsub * S >= bits, bits


def test_restart_segments_follow_the_markers():
    data = encode(make_image("random", 45, 61, 5), 2, restart_marker_blocks=1)
    im = M.Image(data)
    assert im.nseg == im.needed > 1
    for j, (s_off, s_u, q_off, q_u, rst) in enumerate(im.segs):
        assert data[q_off] == 0xFF and s_u <= q_u
        if j + 1 < im.nseg:
            assert rst == j % 8 and data[q_off + 1] == 0xD0 + rst and im.segs[j + 1][0] == q_off + 2


def test_truncated_data_is_an_error_in_the_model():
    data = encode(make_image("random", 45, 61, 5), 2)
    d = JO.parse(data)
    cut = data[: d["scan_begin"] + (len(data) - d["scan_begin"]) // 2]
    assert M.decode(cut)["err"]
    with pytest.raises(JO.CorruptData):
        JO.entropy_decode(cut, JO.parse(cut), JO.geometry(JO.parse(cut)))
