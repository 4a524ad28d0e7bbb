"""CPU: the oracle in every engine layout tests/layout_cases.py names -- lanes in any order, up to 8 of them, groups of 1
to 16 members that include lanes outside the group and remote nodes -- under the adversarial schedules of
tests/fuzz.py: Paxos safety, decisions where the layout is meant to reach, two oracles in lock step; and the input
rules gpx_engine_create / gpx_create_groups / gpx_load_rows share with the engine."""
import numpy as np
import pytest

from fuzz import Fuzzer
from helpers import abi
from layout_cases import LAYOUTS, MAX_MSETS, assert_reached, check_input_rules, mset_limit_engine


@pytest.mark.parametrize("name", sorted(LAYOUTS))
@pytest.mark.parametrize("seed", [1, 2])
def test_oracle_safe_in_every_layout(oracle_lib, name, seed):
    f = Fuzzer([oracle_lib], G=128, W=8, seed=seed, **LAYOUTS[name])
    assert f.run(steps=50, fused_prob=0.3, round_prob=0.4, prepares=True) > 100
    assert_reached(f, name)
    f.close()


@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_two_oracles_in_lock_step(oracle_lib, name):
    """every output of every call, the rows of every lane, flags, ring heads and counters of two oracles"""
    f = Fuzzer([oracle_lib, oracle_lib], G=96, W=4, seed=7, **LAYOUTS[name])
    f.run(steps=40, check_every=5, fused_prob=0.5, round_prob=0.3, round_fn="round_phases", prepares=True)
    f.close()


def test_input_rules_of_the_oracle(oracle_lib):
    check_input_rules(oracle_lib)


def test_member_set_limit_of_the_oracle(oracle_lib):
    e = mset_limit_engine(oracle_lib)
    rows = e.dump_rows(np.arange(MAX_MSETS - 1, MAX_MSETS + 2), 0)
    assert rows["state"].tolist() == [abi.ST_ACTIVE_1, abi.ST_ACTIVE_1, abi.ST_ACTIVE_1]
    e.close()
