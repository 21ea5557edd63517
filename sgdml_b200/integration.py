"""Drop-in of the engine behind the reference's own command line (north_star: "a drop-in behind the existing
CLI"; INTEGRATION.md section 4 realised at run time instead of as a source patch).

The reference's CLI (sgdml/cli.py) instantiates the two classes it imported at module level --
``GDMLTrain`` (cli.py:901, 981, 1221, 1242, 1474) and ``GDMLPredict`` (cli.py:1502) -- and otherwise only moves
task / model dictionaries and ``.npz`` files around.  ``install_into_reference`` rebinds those two names to
the engine's classes.  Task creation and sampling are host-side code that is out of scope for the engine (SURVEY.md
section 2 row 12): the installed training class borrows those methods from the reference's own class, unchanged.

Permutation discovery, which ``create_task`` runs on up to 1000 training geometries (train.py:562-585), is the
exception: its pairwise matching is a GPU workload (``sgdml_b200.perm``).  ``create_task`` looks ``perm.find_perms`` up
in the reference's ``utils.perm`` module when it runs (train.py:72, 578), so that one name is rebound to the engine's
``find_perms`` -- when a CUDA device is visible and the package has such a module; otherwise the reference's own
function stays in place.
"""


def install_into_reference(ref_pkg=None):
    """Rebinds ``sgdml.cli.GDMLTrain`` / ``sgdml.cli.GDMLPredict`` (and the names the training module itself uses for
    its predictor, train.py:1136) to the engine, and ``sgdml.utils.perm.find_perms`` when a device is visible.
    `ref_pkg`: the imported reference package (default: import ``sgdml``).  Returns (train_class, predict_class)."""
    import importlib

    from . import GDMLPredict, GDMLTrain

    ref = ref_pkg if ref_pkg is not None else importlib.import_module('sgdml')
    ref_cli = importlib.import_module(ref.__name__ + '.cli')
    ref_train = importlib.import_module(ref.__name__ + '.train')
    RefTrain = ref_train.GDMLTrain

    class GDMLTrainB200(GDMLTrain):
        """Engine training class with the reference's host-side task functions (train.py:383-724)."""

        create_task = RefTrain.create_task
        create_task_from_model = RefTrain.create_task_from_model
        draw_strat_sample = RefTrain.draw_strat_sample

    for name in ('_draw_strat_sample', '_sample_idxs'):  # private helpers, if this version has them
        if hasattr(RefTrain, name):
            setattr(GDMLTrainB200, name, getattr(RefTrain, name))
    GDMLTrainB200.__name__ = 'GDMLTrain'
    ref_cli.GDMLTrain = GDMLTrainB200
    ref_cli.GDMLPredict = GDMLPredict
    _install_find_perms(ref)
    return GDMLTrainB200, GDMLPredict


def _install_find_perms(ref):
    """Rebinds ``<ref>.utils.perm.find_perms`` to the engine's; returns whether it did.  Without a device, or in a
    package without that module, nothing is touched (the engine's matching has no CPU fallback, the reference's has)."""
    import importlib

    from . import _lib
    from .perm import find_perms

    if _lib.lib().sgdml_b200_device_count() < 1:
        return False
    try:
        ref_perm = importlib.import_module(ref.__name__ + '.utils.perm')
    except ImportError:
        return False
    if not hasattr(ref_perm, 'find_perms'):
        return False
    ref_perm.find_perms = find_perms
    return True
