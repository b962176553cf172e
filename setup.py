"""`pip install .` builds the sm_90a libraries in-tree first (nvcc cross-compiles without a GPU);
the preferred developer flow is still `python -c "import __graft_entry__ as g; g.build()"` so the
`.so` files stay inside the repository tree (they travel with the snapshot to the GPU box)."""
import os
import sys

from setuptools import setup
from setuptools.command.build_py import build_py


class BuildWithKernels(build_py):
    def run(self):
        here = os.path.dirname(os.path.abspath(__file__))
        sys.path.insert(0, here)
        try:
            from distributed_torch_horovod_gcp_b200 import build as native
            native.build(verbose=True)
        except Exception as e:  # noqa: BLE001 - a CPU-only install is still usable (Gloo path)
            print(f"[setup] native build skipped: {e}", file=sys.stderr)
        super().run()


setup(cmdclass={"build_py": BuildWithKernels})
