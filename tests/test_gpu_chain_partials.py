"""GPU suite (-m gpu): the resident chain's per-op reduction state (tmac_chain.cuh): the leader's partial-sum buffer, its mbarrier
phase and the split-phase buffer guard.  Sequences whose clusters are active on some ops only, in both op parities, and a sequence
long enough for that state to wrap many times in one launch; both chain forms must give bit-identical rows."""
import numpy as np
import pytest

from seq_util import inputs, mk, run_form, same_bits, step, stream  # noqa: F401 (fixtures)
from test_gpu_chain import check

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def both_forms(oracle, steps, xs, ext, launches=2):
    got = {}
    for name in ("flow", "barrier"):
        _, got[name] = run_form(name, steps, ext, launches=launches)
        check(oracle, steps, xs, got[name], dense=False)
    for i, (a, b) in enumerate(zip(got["flow"], got["barrier"])):
        assert same_bits(a, b), i


def test_alternating_row_counts(oracle, mk):
    """8 row super-blocks (A) and 4 (B): clusters 4..7 are idle on every B op.  The order puts A ops at both op parities."""
    kw = dict(zp=True)
    a, b = mk(1024, 512, 2, seed=91, **kw), mk(512, 512, 2, seed=92, **kw)
    order = [a, b, a, b, b, a, b, a, a, b]
    steps = [step(o, "x0" if i == 0 else i - 1) for i, o in enumerate(order)]
    xs, ext = inputs(np.random.default_rng(12), x0=512)
    both_forms(oracle, steps, xs, ext)


def test_long_sequence_in_one_launch(oracle, mk):
    """72 ops in one launch: every other op reads its predecessor, the rest a fresh input, so values stay in range."""
    kw = dict(zp=True)
    a, b = mk(512, 256, 2, seed=93, **kw), mk(256, 512, 2, seed=94, **kw)
    steps = [step(b, "x0") if i % 2 == 0 else step(a, i - 1) for i in range(72)]
    xs, ext = inputs(np.random.default_rng(13), x0=512)
    both_forms(oracle, steps, xs, ext)
