"""CPU: the acceptance policy of a least-squares solve (engine.settle_ls), which lib.decompose and the pruner's
pipeline share -- which solves it adds after the first one, and the record it returns, on every branch."""
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")

N, K2 = 50, 9
X = torch.zeros(N, 8 * K2)
Y, Y_BIAS = torch.zeros(N, 4), torch.zeros(4)
IDXS = np.array([True, False, True, True, False, True, False, True])  # K' = 5 * 9 = 45 <= N - 1: primal
DUAL_IDXS = np.ones(8, dtype=bool)                                     # K' = 72 > N - 1: dual


class StubEngine:
    """Records the solves settle_ls asks for; they return small CPU tensors."""

    def __init__(self, exact_fail=0, exact_ratio=0.25, kept=3):
        self.calls = []
        self.exact = (torch.full((4, 45), 1.0, dtype=torch.float64), torch.full((4,), 2.0, dtype=torch.float64),
                      torch.tensor([exact_fail], dtype=torch.int32), torch.tensor([exact_ratio], dtype=torch.float64))
        self.truncated = (torch.full((4, 45), 3.0, dtype=torch.float64), torch.full((4,), 4.0, dtype=torch.float64),
                          kept)

    def reconstruct_exact_async(self, *args):
        self.calls.append(("exact",) + args)
        return self.exact

    def reconstruct_truncated(self, *args):
        self.calls.append(("truncated",) + args)
        return self.truncated


def _settle(eng, mode, fail, ratio, idxs=IDXS):
    from cpb200.engine import settle_ls

    return settle_ls(eng, X, Y, Y_BIAS, idxs, K2, mode, fail, ratio)


def _names(eng, idxs=IDXS):
    for call in eng.calls:  # every solve gets the caller's problem, unchanged
        assert call[1] is X and call[2] is Y and call[3] is Y_BIAS and call[4] is idxs and call[5] == K2
    return [call[0] for call in eng.calls]


def test_dual_path_starts_where_the_normal_equations_lose_full_rank():
    from cpb200.engine import ls_dual

    assert not ls_dual(N, IDXS, K2) and ls_dual(N, DUAL_IDXS, K2)
    assert not ls_dual(46, IDXS, K2) and ls_dual(45, IDXS, K2)  # N - 1 = K' is still primal
    assert not ls_dual(10, np.zeros(8, dtype=bool), K2)


@pytest.mark.parametrize("ratio", [0.5, 1e-4, float("nan")])
def test_fp64_statistics_stand_unless_the_cholesky_fails(ratio):
    from cpb200.engine import GRAM_FP64

    eng = StubEngine()
    W, b, rec = _settle(eng, GRAM_FP64, 0, ratio)
    assert _names(eng) == [] and W is None and b is None
    assert rec.keys() == {"pivot_ratio", "verdict"} and rec["verdict"] == "ok"
    assert rec["pivot_ratio"] == ratio or math.isnan(ratio) and math.isnan(rec["pivot_ratio"])


def test_fp64_singular_gets_the_truncated_solution():
    from cpb200.engine import GRAM_FP64

    eng = StubEngine(kept=31)
    W, b, rec = _settle(eng, GRAM_FP64, 1, 1e-13)
    assert _names(eng) == ["truncated"]
    assert W is eng.truncated[0] and b is eng.truncated[1]
    assert rec == {"pivot_ratio": 1e-13, "verdict": "truncated", "rank": 31}


@pytest.mark.parametrize("mode", [0, 1], ids=["fp64", "tc"])
def test_dual_path_is_never_redone(mode):
    eng = StubEngine(kept=40)
    W, b, rec = _settle(eng, mode, 0, 1e-6, idxs=DUAL_IDXS)  # a low ratio alone changes nothing on the dual path
    assert _names(eng, DUAL_IDXS) == [] and W is None and rec == {"pivot_ratio": 1e-6, "verdict": "ok"}
    eng = StubEngine(kept=40)
    W, b, rec = _settle(eng, mode, 1, 1e-14, idxs=DUAL_IDXS)
    assert _names(eng, DUAL_IDXS) == ["truncated"]
    assert W is eng.truncated[0] and b is eng.truncated[1]
    assert rec == {"pivot_ratio": 1e-14, "verdict": "truncated", "rank": 40}


def test_tensor_core_solve_stands_at_the_threshold():
    from cpb200.engine import GRAM_3XTF32, LS_RATIO_MIN

    eng = StubEngine()
    W, b, rec = _settle(eng, GRAM_3XTF32, 0, LS_RATIO_MIN)
    assert _names(eng) == [] and W is None and b is None
    assert rec == {"pivot_ratio": LS_RATIO_MIN, "verdict": "ok"}


@pytest.mark.parametrize("fail,ratio", [(0, 0.0049), (0, float("nan")), (1, 0.3)], ids=["low", "nan", "fail"])
def test_tensor_core_solve_is_redone_from_exact_statistics(fail, ratio):
    from cpb200.engine import GRAM_3XTF32

    eng = StubEngine(exact_ratio=0.125)
    W, b, rec = _settle(eng, GRAM_3XTF32, fail, ratio)
    assert _names(eng) == ["exact"]
    assert W is eng.exact[0] and b is eng.exact[1]
    assert rec.keys() == {"pivot_ratio", "pivot_ratio_exact", "verdict"}
    assert rec["verdict"] == "redo->ok" and rec["pivot_ratio_exact"] == 0.125
    assert rec["pivot_ratio"] == ratio or math.isnan(ratio) and math.isnan(rec["pivot_ratio"])


def test_redo_that_fails_gets_the_truncated_solution():
    from cpb200.engine import GRAM_3XTF32

    eng = StubEngine(exact_fail=1, exact_ratio=1e-13, kept=17)
    W, b, rec = _settle(eng, GRAM_3XTF32, 0, 1e-3)
    assert _names(eng) == ["exact", "truncated"]
    assert W is eng.truncated[0] and b is eng.truncated[1]
    assert rec == {"pivot_ratio": 1e-3, "pivot_ratio_exact": 1e-13, "verdict": "truncated", "rank": 17}
