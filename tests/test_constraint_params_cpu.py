"""The estimators' constraint parameters in the native parameter string: lists and NumPy arrays give the same keys, and an empty value
adds none."""
import numpy as np

from mmlspark_b200.lightgbm import Frame, LightGBMRegressor


def _params(**kw):
    df = Frame({"features": np.zeros((10, 5)), "label": np.zeros(10)})
    return LightGBMRegressor(**kw).getTrainParams(1, df).to_string()


def test_interaction_constraints_from_lists_and_arrays():
    want = "interaction_constraints=[0,1],[1,2,3],[4] "
    assert _params(interactionConstraints=[[0, 1], [1, 2, 3], [4]]).endswith(want)
    assert _params(interactionConstraints=[np.array([0, 1]), np.array([1, 2, 3]), np.array([4])]).endswith(want)
    assert _params(interactionConstraints=np.array([[0, 1], [2, 3]])).endswith("interaction_constraints=[0,1],[2,3] ")
    assert "interaction" not in _params(interactionConstraints=np.zeros((0, 2), int))
    assert "interaction" not in _params()


def test_monotone_constraints_from_an_array():
    want = "monotone_constraints=1,-1,0,0,1 monotone_constraints_method=basic monotone_penalty=0.0 "
    assert _params(monotoneConstraints=[1, -1, 0, 0, 1]).endswith(want)
    assert _params(monotoneConstraints=np.array([1, -1, 0, 0, 1])).endswith(want)
    assert "monotone" not in _params(monotoneConstraints=np.array([], int))
