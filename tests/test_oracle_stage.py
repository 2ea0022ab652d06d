"""oracle/stage_ref.installed(), the context every runner of the staged reference code uses: what it puts in place is undone on exit,
also when the body raises.  No GPU, no staged reference needed."""
import os
import sys
import types

import pytest

from oracle import stage_ref


def test_installed_restores_everything_when_the_body_raises(tmp_path):
    replaced, removed, added = "_pcb_stage_replaced", "_pcb_stage_removed", "_pcb_stage_added"
    originals = {replaced: types.ModuleType(replaced), removed: types.ModuleType(removed)}
    sys.modules.update(originals)
    path, cwd, argv = list(sys.path), os.getcwd(), sys.argv
    stand_in = types.ModuleType(replaced)
    (tmp_path / "elsewhere").mkdir()
    try:
        with pytest.raises(RuntimeError, match="raised inside"):
            with stage_ref.installed({replaced: stand_in, removed: None, added: None}, path=[str(tmp_path)], cwd=tmp_path,
                                     argv=["script.py", "--flag"]):
                assert sys.modules[replaced] is stand_in and removed not in sys.modules
                assert sys.path[:len(path) + 1] == [str(tmp_path)] + path
                assert os.path.samefile(os.getcwd(), tmp_path) and sys.argv == ["script.py", "--flag"]
                sys.modules[added] = types.ModuleType(added)        # as a staged module imported inside would be
                sys.path.append(str(tmp_path / "appended"))         # as staged code that extends sys.path does
                os.chdir("elsewhere")
                raise RuntimeError("raised inside")
        assert sys.modules[replaced] is originals[replaced] and sys.modules[removed] is originals[removed]
        assert added not in sys.modules
        assert sys.path == path and os.getcwd() == cwd and sys.argv is argv
    finally:
        for k in (replaced, removed, added):
            sys.modules.pop(k, None)
