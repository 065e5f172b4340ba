"""CPU: the shared gather-test scaffolding's patch of the oracle's CD solver, which is process-wide state."""
import numpy as np
import pytest

import cp_oracle as O
import gather_checks as GC


def test_seeded_lasso_feeds_each_solver_the_seeds_and_restores_lasso_init_on_an_exception():
    orig = O.LassoCD.__init__
    with pytest.raises(RuntimeError, match="inside"):
        with GC.seeded_lasso(np.array([5, 7])):
            a, b = O.LassoCD(alpha=1e-3), O.LassoCD(alpha=1e-3)
            assert [a.rng.randint(0, 10), a.rng.randint(0, 10), b.rng.randint(0, 10)] == [5, 7, 5]
            raise RuntimeError("inside")
    assert O.LassoCD.__init__ is orig
    assert O.LassoCD(alpha=1e-3).rng is np.random.mtrand._rand
