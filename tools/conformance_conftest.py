"""conftest used by tools/run_reference_tests.sh: aliases `pypose` to pypose_b200 (CPU, oracle-backed test kernels)."""
import importlib
import os
import sys

sys.path.insert(0, os.environ['PYPOSE_B200_ROOT'])
import tests.conftest  # noqa: F401,E402
import pypose_b200  # noqa: E402

sys.modules['pypose'] = pypose_b200
for m in ('optim', 'module', 'func', 'testing', 'lietensor', 'function', 'basics', 'autograd', 'optim.solver',
          'optim.strategy', 'optim.scheduler', 'optim.kernel', 'optim.corrector', 'optim.functional',
          'optim.optimizer', 'lietensor.lietensor', 'autograd.function'):
    sys.modules[f'pypose.{m}'] = importlib.import_module(f'pypose_b200.{m}')
