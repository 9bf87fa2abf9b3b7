"""H100-native RBM/DBM engine behind the yell/boltzmann-machines Python API.

Host side: thin Python (this package).  Compute: hand-written sm_90a CUDA in
``../csrc`` reached through the C-ABI of ``include/bm.h`` (``libbm.so``).
"""
from . import base
from . import utils
from . import layers
from . import ebm
from . import rbm
from .rbm import BaseRBM, BernoulliRBM, MultinomialRBM, GaussianRBM, ClassificationRBM, logit_mean, fit_many
from . import dbm
from .dbm import DBM
from . import class_dbm
from .class_dbm import ClassificationDBM
