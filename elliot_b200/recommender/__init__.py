"""Model registry: the class names the reference resolves from the YAML model key
(elliot/run.py:75, elliot/recommender/__init__.py)."""
from .bprmf import BPRMF, MFModel  # noqa: F401
from .bprmf_batch import BPRMF_batch, BPRMFBatchModel  # noqa: F401
from .multi_vae import MultiVAE, VariationalAutoEncoder  # noqa: F401
from .neumf import NeuMF, NeuralMatrixFactorizationModel  # noqa: F401
from .mf2020 import MF2020, MF2020Model  # noqa: F401
from .multi_dae import MultiDAE, DenoisingAutoEncoder  # noqa: F401
from .gmf import GMF, GeneralizedMatrixFactorizationModel  # noqa: F401
from .knn import ItemKNN, UserKNN, KNNModel  # noqa: F401
from .als import iALS, WRMF, ALSModel  # noqa: F401
from .ease import EASER, EASEModel  # noqa: F401
from .rp3beta import RP3beta, RP3Model  # noqa: F401
from .slim import Slim, SlimModel  # noqa: F401
from .pure_svd import PureSVD, PureSVDModel  # noqa: F401
