"""sgdml_b200 -- H100-native engine for sGDML's two dense hot paths (SURVEY.md section 8):
(a) Hessian-kernel matrix assembly + FP64 Cholesky solve behind ``GDMLTrain.train(task)``,
(b) batched energy/force prediction behind ``GDMLPredict(model).predict(R)``.

Host code is Python; all arithmetic runs in hand-written sm_90a CUDA kernels behind the C
ABI declared in ``include/sgdml_b200.h`` (``sgdml_b200/libsgdml_b200.so``).  There is no
CPU fallback.
"""

__version__ = '0.1.0'

from .md import (GDMLIRC, GDMLNEB, GDMLDimer, GDMLDynamics, GDMLMetadynamics, GDMLNPTDynamics,  # noqa: F401
                 GDMLPathIntegralDynamics, GDMLRelaxation, GDMLReplicaExchange, GDMLUmbrellaSampling)
from .perm import find_perms  # noqa: F401
from .posterior import GDMLPosterior  # noqa: F401
from .predict import GDMLPredict  # noqa: F401
from .train import GDMLTrain  # noqa: F401
from .vib import GDMLVibrations, harmonic_rate, thermo  # noqa: F401
