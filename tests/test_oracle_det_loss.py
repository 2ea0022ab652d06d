"""oracle/det_loss_cpu.py against the original `loss_helper.get_loss` run unmodified in fp64 (tests/golden/detection_loss.npz, written by
tests/golden/make_detection_loss_golden.py): the assignments, objectness labels and masks exactly -- planted ties, a padded-slot
assignment, gray-zone proposals and a scene with no positive proposal included -- and the 13 outputs and the gradients of `loss` to
fp64 rounding."""
import os

import numpy as np
import pytest

from oracle import det_loss_cpu as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "detection_loss.npz")
DATASETS = {"scannet": (1, 18, 18), "sunrgbd": (12, 10, 10)}        # NH, NS, C
CASES = [f"{d}_v{v}" for d in DATASETS for v in (1, 3)]
GRAD_INPUTS = ("vote_xyz", "seed_xyz", "center", "objectness_scores", "heading_scores", "heading_residuals_normalized", "size_scores",
               "size_residuals_normalized", "sem_cls_scores")


def golden(name):
    """(end_points numpy dict, mean_size, (NH, NS, C), the original's results) of one golden case."""
    z = np.load(GOLDEN)
    ep = {k.split("/")[2]: z[k] for k in z.files if k.startswith(name + "/in/")}
    out = {k.split("/")[2]: z[k] for k in z.files if k.startswith(name + "/out/")}
    return ep, z[name + "/mean_size"], DATASETS[name.rsplit("_", 1)[0]], out


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_original(name):
    ep, ms, (NH, NS, C), want = golden(name)
    r = O.forward(ep, ms, NH, C)
    for k in ("objectness_label", "objectness_mask", "object_assignment"):
        assert np.array_equal(r[k], want[k]), k
    for k in O.OUTPUTS:
        assert abs(r[k] - float(want[k])) <= 1e-12 * max(1.0, abs(float(want[k]))), (k, r[k], float(want[k]))
    g = O.backward(ep, r, np.eye(len(O.OUTPUTS))[O.OUTPUTS.index("loss")], ms, NH)
    for k in GRAD_INPUTS:
        np.testing.assert_allclose(g[k], want["grad_" + k], rtol=0, atol=1e-12, err_msg=k)


def test_golden_holds_the_planted_cases():
    for name in CASES:
        ep, *_, want = golden(name)
        a, lab, m = want["object_assignment"], want["objectness_label"], want["objectness_mask"]
        assert a[0, 0] == 0 and lab[0, 0] == 1                      # the tie between slots 0 and 1 goes to 0
        assert a[0, 1] >= ep["box_label_mask"][0].sum()             # a padded zero slot
        assert m[0, 2] == 0 and m[0, 3] == 0                        # gray zone
        assert lab[1].sum() == 0                                    # no positive proposal in scene 1
        g = want["grad_vote_xyz"]
        V = ep["vote_xyz"].shape[1] // ep["seed_xyz"].shape[1]
        assert (g[0, V] == 0).all()                                 # a vote exactly on its GT vote: |x|'(0) = 0
