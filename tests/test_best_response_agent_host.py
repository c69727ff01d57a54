"""Best response as an agent, host side: the tie rule of the one-hot tables and the size rule that refuses a spec whose
best-response tables cannot fit (no GPU needed)."""
import numpy as np
import pytest
import torch

from pokerrl_b200.board_engine import best_response_bytes, check_best_response_fits, first_max_onehot

CLASSES, DEALS = 134459, 2598960


def test_table_bytes_of_the_full_game():
    rows_deep, rows_short = 14, 8
    pos_hand = CLASSES * 1081 * 2
    assert best_response_bytes(CLASSES, rows_deep) == CLASSES * rows_deep * 4352 + pos_hand
    assert round(CLASSES * rows_deep * 4352 / 1e9, 2) == 8.19
    assert round(CLASSES * rows_short * 4352 / 1e9, 2) == 4.68
    assert round(pos_hand / 1e6) == 291
    assert round(best_response_bytes(DEALS, rows_deep) / 1e9) == 164  # 158 GB of rows + 5.6 GB of pos_hand
    assert round(DEALS * rows_deep * 4352 / 1e9) == 158
    assert round(DEALS * rows_short * 4352 / 1e9) == 90


def test_an_oversized_spec_is_refused_with_the_byte_count():
    need = best_response_bytes(DEALS, 14)
    with pytest.raises(ValueError, match="%d bytes" % need):
        check_best_response_fits(need, 80 * 10 ** 9)
    check_best_response_fits(best_response_bytes(CLASSES, 14), 80 * 10 ** 9)


def test_onehot_takes_the_first_maximum_like_np_argmax():
    rng = np.random.default_rng(3)
    v = rng.integers(0, 3, size=(5, 4, 200)).astype(np.float32)  # many ties
    v[:, :, :10] = 7.0  # all children tied
    for dim in (0, 1, 2):
        got = first_max_onehot(torch.from_numpy(v), dim).numpy()
        want = np.moveaxis(np.eye(v.shape[dim], dtype=np.float32)[np.argmax(v, axis=dim)], -1, dim)
        assert np.array_equal(got, want), dim
    x = torch.tensor([[1.0, -float("inf")], [1.0, 2.0], [0.5, 2.0]])
    assert torch.equal(first_max_onehot(x, 0), torch.tensor([[1.0, 0.0], [0.0, 1.0], [0.0, 0.0]]))
