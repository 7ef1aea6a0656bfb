"""Pin the CPU oracle against golden vectors minted from the unmodified reference at embedding widths 32, 96 and 192
(tests/golden/make_golden_width.py), at the tolerances of tests/test_oracle_golden.py."""
import pytest

from tests import test_oracle_golden as OG

WIDTH_CASES = ("width_d32_train_rand_k3", "width_d96_train_empty_k2", "width_d192_eval_alias_k2")


@pytest.mark.parametrize("case", WIDTH_CASES)
@pytest.mark.parametrize("variant", ["literal", "closed"])
def test_forward_losses_grads(case, variant):
    OG.test_forward_losses_grads(case, variant)


@pytest.mark.parametrize("case", WIDTH_CASES)
def test_infonce_block_independent(case):
    OG.test_infonce_block_independent(case)


def test_cases_cover_the_new_widths():
    from tests.golden_util import Golden
    assert sorted(Golden(c).cfg["d"] for c in WIDTH_CASES) == [32, 96, 192]
