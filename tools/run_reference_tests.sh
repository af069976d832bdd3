#!/bin/bash
# API conformance: run the REFERENCE's own tests (tests/lietensor, tests/basics, tests/optim, tests/module/test_loss.py,
# test_pnp.py, test_dynamics.py, test_lqr.py, test_mpc.py)
# against pypose_b200.
# Needs a pypose v0.9.5 checkout named by PYPOSE_REFERENCE; the tests are copied to a scratch dir, never into the repo.
# Deselected: test_sparse_lm.py (needs CUDA + the external `bae` package), test_parameter_dispatch (monkeypatches
# the reference's private bae loader), the three EPnP tests that download their data (no network; the 6-point test runs).  Known remaining failure: test_quat2unit before convert.quat2unit existed.
set -e
REF=${PYPOSE_REFERENCE:?set PYPOSE_REFERENCE to a pypose v0.9.5 checkout}
export PYPOSE_B200_ROOT=$(cd "$(dirname "$0")/.." && pwd)
D=$(mktemp -d)
cp $PYPOSE_B200_ROOT/tools/conformance_conftest.py $D/conftest.py
cp -r $REF/tests/lietensor $REF/tests/basics $REF/tests/optim $D/
mkdir -p $D/module $D/function && cp $REF/tests/module/test_loss.py $REF/tests/module/test_pnp.py $REF/tests/module/test_dynamics.py $REF/tests/module/test_lqr.py $REF/tests/module/test_mpc.py $D/module/ && cp $REF/tests/function/test_spline.py $REF/tests/function/test_checking.py $D/function/
cd $D && PYTHONDONTWRITEBYTECODE=1 python -m pytest lietensor basics optim module function -q -p no:cacheprovider \
    --deselect optim/test_sparse_lm.py --deselect lietensor/test_lietensor.py::test_parameter_dispatch \
    --deselect module/test_pnp.py::TestEPnP::test_epnp_nonbatch --deselect module/test_pnp.py::TestEPnP::test_epnp_highdim \
    --deselect module/test_pnp.py::TestEPnP::test_epnp_random "$@"
