"""tests/golden/reference.py as the one way to the reference's Python: every golden generator's import, called in one process, leaves
sys.path and the top-level module names the reference's files import as it found them, so no test depends on which generator ran
before it; and no other Python file reads the reference root's variable or reaches the stand-ins through a path."""
import os
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import reference  # noqa: E402

NAMES = {"lietorch", "torch_scatter", "droid_backends", "geom", "modules", "factor_graph", "depth_video", "motion_filter",
         "trajectory_filler", "droid_async", "align"}


@pytest.mark.skipif(not reference.present("droid_slam"), reason="reference tree not present")
def test_every_generator_import_leaves_sys_path_and_sys_modules_alone():
    import make_async_golden
    import make_ba_layer_golden
    import make_corr_training_golden
    import make_encoder_golden
    import make_factor_graph_golden
    import make_motion_filter_golden
    import make_proximity_golden
    import make_reference_python_golden
    import make_trajectory_filler_golden
    import make_update_golden
    importers = {"reference_python": make_reference_python_golden.import_reference,
                 "proximity": make_proximity_golden.import_reference_factor_graph,
                 "factor_graph": make_factor_graph_golden.import_reference_factor_graph,
                 "motion_filter": make_motion_filter_golden.import_reference,
                 "trajectory_filler": make_trajectory_filler_golden.import_reference_trajectory_filler,
                 "async": make_async_golden.import_reference,
                 "ba_layer": make_ba_layer_golden.import_reference_ba,
                 "corr_training": make_corr_training_golden.import_reference,
                 "encoder": make_encoder_golden.import_reference,
                 "update": make_update_golden.import_reference}
    for name, importer in importers.items():
        path, before = list(sys.path), set(sys.modules)
        assert importer() is not None, name
        assert sys.path == path, name
        added = {m for m in set(sys.modules) - before if m.split(".")[0] in NAMES}
        assert not added, (name, sorted(added))


def test_only_reference_py_reads_the_root_or_puts_the_stand_ins_on_sys_path():
    offenders = []
    for top in ("tests", "oracle", "tools"):
        for dirpath, dirs, files in os.walk(os.path.join(ROOT, top)):
            dirs[:] = [d for d in dirs if d not in ("_ref", "__pycache__")]
            for f in files:
                p = os.path.join(dirpath, f)
                if not f.endswith(".py") or p in (reference.__file__, os.path.abspath(__file__)):
                    continue
                with open(p) as fh:
                    src = fh.read()
                if "DROID_REFERENCE_ROOT" in src or re.search(r"""shims["']""", src):
                    offenders.append(os.path.relpath(p, ROOT))
    assert not offenders, offenders
