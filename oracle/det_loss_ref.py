"""Stages the original VoteNet network heads next to the oracle, so that the GPU tests and profiles/bench_det_loss.py can build the
original `VoteNet` on this library's backbone and compare its training step under the original criterion and pointcontrast_b200.det_loss:

    python oracle/det_loss_ref.py       (also run by __graft_entry__.build(), after oracle/detection_ref.py and oracle/det_eval_ref.py,
                                         which both clear parts of oracle/_ref/votenet/)

Copies, byte for byte, `models/{votenet,voting_module,proposal_module}.py` from `<root>/downstream/votenet_det_new/` into
`oracle/_ref/votenet/models/` (git-ignored); the criterion itself, `models/loss_helper.py` with `lib/utils/nn_distance.py`, is staged by
oracle/det_eval_ref.py.  <root> is $PCB_REFERENCE_ROOT, with the same default as oracle/stage_ref.py; where the original is absent
nothing is staged.  Nothing under pointcontrast_b200/ imports this.
"""
import os
import shutil

SRC = os.path.join(os.environ.get("PCB_REFERENCE_ROOT", "/root/reference"), "downstream", "votenet_det_new", "models")
DST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "votenet", "models")
FILES = ("votenet.py", "voting_module.py", "proposal_module.py")


def stage(verbose=False):
    if not os.path.isfile(os.path.join(SRC, "votenet.py")) or not os.path.isdir(DST):
        return False
    for f in FILES:
        shutil.copyfile(os.path.join(SRC, f), os.path.join(DST, f))
    if verbose:
        print("staged", SRC, "(VoteNet heads) ->", DST)
    return True


def available():
    return all(os.path.isfile(os.path.join(DST, f)) for f in FILES)


if __name__ == "__main__":
    print("staged" if stage(True) else f"{SRC} not present (or the backbone is not staged): nothing staged")
