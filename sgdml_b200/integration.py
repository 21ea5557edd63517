"""Drop-in of the engine behind the reference's own command line (north_star: "a drop-in behind the existing
CLI"; INTEGRATION.md section 4 realised at run time instead of as a source patch).

The reference's CLI (sgdml/cli.py) instantiates the two classes it imported at module level --
``GDMLTrain`` (cli.py:901, 981, 1221, 1242, 1474) and ``GDMLPredict`` (cli.py:1502) -- and otherwise only moves
task / model dictionaries and ``.npz`` files around.  ``install_into_reference`` rebinds those two names to
the engine's classes.  Task creation, sampling and permutation discovery are host-side code that is out of
scope for the engine (SURVEY.md section 2 rows 12-13): the installed training class borrows those methods from
the reference's own class, unchanged.
"""


def install_into_reference(ref_pkg=None):
    """Rebinds ``sgdml.cli.GDMLTrain`` / ``sgdml.cli.GDMLPredict`` (and the names the training module itself uses for
    its predictor, train.py:1136) to the engine.  `ref_pkg`: the imported reference package (default: import
    ``sgdml``).  Returns (train_class, predict_class)."""
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
    return GDMLTrainB200, GDMLPredict
