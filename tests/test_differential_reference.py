"""Differential tests of the Python drop-in surface against the UNMODIFIED reference modules, on seeded randomised
inputs.  The reference's results were recorded once by oracle/gen_golden.py (tests/golden/reference_digests.json:
the SHA-256 of each case's canonical form, tests/reference_cases.py); here the same cases run against qrec_b200 and
must give exactly the same results.  Nothing here is imported by the product."""
import numpy as np
import pytest

import reference_cases as RC


@pytest.fixture(scope='module')
def mine():
    return RC.qrec_b200_modules()


def _check(name, mine, tmp_path):
    assert RC.digest(RC.CASES[name](mine, str(tmp_path))) == RC.recorded(name), name


def test_option_conf_equals_reference_on_random_strings(mine, tmp_path):
    _check('option_conf', mine, tmp_path)


def test_model_conf_equals_reference(mine, tmp_path):
    _check('model_conf', mine, tmp_path)
    from qrec_b200.util.config import ModelConf
    bad = tmp_path / 'bad2.conf'
    bad.write_text('a=1\nnot a pair\nb=2=3\n\nc=x y\n')
    assert ModelConf(str(bad)).config == {'a': '1', 'c': 'x y'}


def test_measures_equal_reference_on_random_rankings(mine, tmp_path):
    _check('measures', mine, tmp_path)


def test_find_k_largest_equals_reference_numba_heap(mine, tmp_path):
    _check('find_k_largest', mine, tmp_path)


def test_rating_equals_reference_on_random_data(mine, tmp_path):
    _check('rating', mine, tmp_path)


def test_data_split_and_cv_equal_reference(mine, tmp_path):
    _check('data_split', mine, tmp_path)


def test_loader_equals_reference_on_shipped_datasets(mine, tmp_path):
    _check('loader', mine, tmp_path)


def test_eval_ranking_and_lr_schedule_equal_reference(mine, tmp_path):
    """Recommender.evalRanking / IterativeRecommender.isConverged of the mirror classes against the reference
    classes, both fed the same numpy P, Q: identical recommendation lines, metric strings, learning-rate updates
    and generator state."""
    _check('eval_ranking', mine, tmp_path)


@pytest.mark.parametrize('seed', [0, 7, 2024])
def test_minibatch_samplers_equal_reference_on_random_data(mine, tmp_path, seed):
    """DeepRecommender.next_batch_pairwise / next_batch_pointwise (C MT19937 clone underneath) against the reference
    generators (Python `random`) on random interaction lists with duplicates and non-binary ratings: every batch,
    the shuffled list and the generator state afterwards."""
    got = RC.CASES['minibatch_samplers_%d' % seed](mine, str(tmp_path))
    assert len(got[0]) == 8 and len(got[0][-1][0]) == 1000 - 7 * 128
    assert RC.digest(got) == RC.recorded('minibatch_samplers_%d' % seed)


def test_interaction_table_equals_reference_loader_and_rating(tmp_path):
    """f-3: the array-backed table built from the shipped FilmTrust file has the reference's id space."""
    from qrec_b200.data.interactions import InteractionTable
    t = InteractionTable.from_text(RC.ratings_file(str(tmp_path)), binarize_threshold=1.0)
    assert len(t) == 34437
    got = [len(t), t.user_names.tolist(), t.item_names.tolist(), np.asarray(t.u).tolist(), np.asarray(t.i).tolist()]
    assert RC.digest(got) == RC.recorded('interaction_table_ids')
