"""The engine as a drop-in behind the reference's own CLI (INTEGRATION.md section 4), checked against what the unmodified
reference recorded in tests/golden/dropin/ (make_golden.py dropin): the parameter lists of its GDMLTrain / GDMLPredict
entry points, and a task made by its create_task with the model its GDMLTrain.train makes of it.  The rebinding of
`install_into_reference` is checked on a stub package shaped like the reference (a `cli` and a `train` module)."""

import json
import os
import sys
import types

import numpy as np
import pytest

from conftest import GOLDEN_DIR, rel_err

DROPIN_DIR = os.path.join(GOLDEN_DIR, 'dropin')


def _reference():
    with open(os.path.join(DROPIN_DIR, 'reference_model.json')) as f:
        return json.load(f)


def _params(f):
    import inspect

    return list(inspect.signature(f).parameters)


def _stub_reference(monkeypatch):
    """A package `refstub` with the two modules install_into_reference touches: `cli` (module-level GDMLTrain /
    GDMLPredict names) and `train` (a GDMLTrain owning the host-side task functions the engine borrows)."""

    class RefTrain(object):
        def create_task(self, *a, **k):
            return 'task'

        def create_task_from_model(self, *a, **k):
            return 'task from model'

        def draw_strat_sample(self, *a, **k):
            return 'sample'

    pkg = types.ModuleType('refstub')
    cli = types.ModuleType('refstub.cli')
    train = types.ModuleType('refstub.train')
    cli.GDMLTrain, cli.GDMLPredict = RefTrain, object
    train.GDMLTrain = RefTrain
    pkg.cli, pkg.train = cli, train
    for name, mod in (('refstub', pkg), ('refstub.cli', cli), ('refstub.train', train)):
        monkeypatch.setitem(sys.modules, name, mod)
    return pkg, RefTrain


def test_install_rebinds_reference_cli_and_signatures_match(monkeypatch):
    """CPU: the two names the reference CLI instantiates are rebound, the task functions are borrowed from the
    reference's class unchanged, and the constructor / train / predict parameter lists of the engine classes equal the
    reference's (train.py:306, 836-841; predict.py:249-258, 1146)."""
    import sgdml_b200
    from sgdml_b200.integration import install_into_reference

    pkg, RefTrain = _stub_reference(monkeypatch)
    T, P = install_into_reference(pkg)
    assert pkg.cli.GDMLTrain is T and pkg.cli.GDMLPredict is P
    assert issubclass(T, sgdml_b200.GDMLTrain) and P is sgdml_b200.GDMLPredict
    for name in ('create_task', 'create_task_from_model', 'draw_strat_sample'):
        assert getattr(T, name) is getattr(RefTrain, name)

    sig = _reference()['signatures']
    assert _params(T.__init__) == sig['GDMLTrain.__init__']
    assert _params(T.train) == sig['GDMLTrain.train']
    assert _params(P.__init__) == sig['GDMLPredict.__init__']
    assert _params(P.predict)[:3] == sig['GDMLPredict.predict'][:3]


@pytest.mark.gpu
def test_train_reference_task_matches_reference_model():
    """GDMLTrain.train on a task made by the reference's own create_task: the model dict has the reference model's
    keys, shapes and dtypes, its c and std, and predicts what the reference-trained model predicts (1e-6 rel)."""
    import sgdml_b200

    ref = _reference()
    with np.load(os.path.join(DROPIN_DIR, 'reference_task.npz'), allow_pickle=False) as f:
        task = {k: f[k] for k in f.files}
    Rq = task.pop('R_query')
    model = sgdml_b200.GDMLTrain().train(task)
    assert sorted(model.keys()) == ref['model_keys']
    for k in ('R_desc', 'R_d_desc_alpha', 'alphas_F', 'perms', 'tril_perms_lin'):
        assert list(np.asarray(model[k]).shape) == ref['model_shapes'][k], k
    for k in ('R_desc', 'R_d_desc_alpha', 'alphas_F', 'perms', 'tril_perms_lin', 'sig', 'c', 'std', 'solver_name'):
        assert str(np.asarray(model[k]).dtype) == ref['model_dtypes'][k], k
    assert str(model['solver_name']) == 'analytic'
    assert abs(float(model['c']) - ref['c']) < 1e-6 * abs(ref['c'])
    assert abs(float(model['std']) - ref['std']) < 1e-12 * ref['std']
    E, F = sgdml_b200.GDMLPredict(model).predict(Rq)
    assert rel_err(E, ref['E_query']) < 1e-6
    assert rel_err(F, ref['F_query']) < 1e-6
