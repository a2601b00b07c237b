"""CPU oracle for the dense-BA update hot path of DROID-SLAM.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is imported by the product package
(``droid_slam_b200``); only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` may import it, and only as the checker.

The oracle is a vectorised PyTorch (CPU) restatement of the reference's CUDA kernels
(``/root/reference/src/*.cu``), quirks included (SURVEY.md section 8a, Q1-Q12).  Each function cites the
reference file:line it follows.

Parity pinning: the reference ships NO golden vectors or unit tests for this path (SURVEY.md
section 4 / 8c).  The oracle is pinned instead against the reference's own CUDA build run on a
H100 (``oracle/build_ref.sh`` -> ``oracle/_ref/droid_backends_ref``; fixtures under
``tests/golden/`` made by ``tests/golden/make_golden.py``) -- see DESIGN.md "Oracle pinning".
"""
from .se3 import *      # noqa: F401,F403
from .geom import *     # noqa: F401,F403
from .ba import *       # noqa: F401,F403
from .corr import *     # noqa: F401,F403
from .update import *   # noqa: F401,F403
from .upsample import *  # noqa: F401,F403
