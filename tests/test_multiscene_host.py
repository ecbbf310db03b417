"""Host logic of scene-batched sampling: the row schedule of PLMSSampler.sample_rows and KeyedNoise serving a prefix of its rows."""
import pytest
import torch

from sparsefusion_b200.plms import _row_lin, _step_scalars, row_schedule

MAX_THRES = [0.004, 0.013, 0.13, 0.37, 0.62, 0.99]


def test_row_schedule_of_six_noise_levels():
    s = row_schedule(MAX_THRES, 50)
    assert s.n_steps == [0, 1, 13, 37, 50, 50]
    assert s.calls == [0, 2, 14, 38, 51, 51]             # the single-row sampler's n + 1 evaluations (none for n = 0)
    assert s.order == [4, 5, 3, 2, 1, 0]                 # descending n, stable
    assert s.rounds == 51                                # one UNet evaluation + one update launch per round
    # active rows per round: rounds 0 and 1 are step 0 (e_t, then e_next), round j >= 2 is step j - 1
    want = [5, 5] + [4] * 12 + [3] * 24 + [2] * 13
    assert s.batch == want
    for k in range(6):                                   # a row's evaluations = rounds it is active in
        p = s.order.index(k)
        assert sum(1 for b in s.batch if p < b) == s.calls[k]


def test_row_schedule_scalars_are_each_rows_own():
    s = row_schedule(MAX_THRES, 50)
    for j in range(s.rounds):
        step = max(j - 1, 0)
        for p in range(6):
            if p < s.batch[j]:
                lin = _row_lin(MAX_THRES[s.order[p]], 50)
                assert s.scalars[j][p] == _step_scalars(lin[step], lin[step + 1])
                assert s.levels[s.level_idx[j][p]] == (lin[1] if j == 1 else lin[step])
            else:
                assert s.scalars[j][p] == (0.0,) * 5
    assert len(set(s.levels)) == len(s.levels)


def test_row_schedule_of_one_shared_level_is_the_single_run():
    for m in (0.004, 0.13, 0.62, 0.995):
        s = row_schedule([m] * 3, 50)
        lin = _row_lin(m, 50)
        assert s.order == [0, 1, 2] and s.levels == (lin if len(lin) > 1 else [])
        assert s.rounds == (len(lin) if len(lin) > 1 else 0) and all(b == 3 for b in s.batch)
        assert all(len(set(idx)) == 1 for idx in s.level_idx)


def test_keyed_noise_serves_a_prefix_of_rows():
    from sparsefusion_b200.distillation import KeyedNoise
    like = torch.empty(3, 4, 2, 2)
    full = KeyedNoise([5, 6, 7], 'cpu')
    part = KeyedNoise([5, 6, 7], 'cpu')
    a = [full(like) for _ in range(4)]
    b = [part(like), part(like[:2], rows=[2, 0]), part(like[:2], rows=[0, 2]), part(like[:1], rows=[2])]
    assert torch.equal(a[0], b[0])
    assert torch.equal(b[1], a[1][[2, 0]]) and torch.equal(b[2], a[2][[0, 2]]) and torch.equal(b[3], a[3][[2]])
    with pytest.raises(AssertionError):
        part(like[:1], rows=[1])                       # row 1 left the run: it may not draw again
