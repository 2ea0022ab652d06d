"""The original VoteNet network heads (`models/{votenet,voting_module,proposal_module}.py`), staged by oracle/stage_ref.py under
`oracle/_ref/votenet/models/` beside the backbone (oracle/detection_ref.py) and the criterion (`models/loss_helper.py`, see
oracle/det_eval_ref.py), so that the GPU tests and profiles/bench_det_loss.py can build the original `VoteNet` on this library's
backbone and compare its training step under the original criterion and pointcontrast_b200.det_loss.  Nothing under
pointcontrast_b200/ imports this.
"""
from oracle import stage_ref


def available():
    return stage_ref.available("votenet")
