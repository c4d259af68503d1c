"""3dunetcnn_b200 -- H100-native (sm_90a) 3D U-Net forward/backward path behind the reference's model / loss / train /
predict interface.  The directory name starts with a digit, so import it with
``importlib.import_module("3dunetcnn_b200")`` (tests/conftest.py and __graft_entry__.py do).
"""
from . import lib, models, losses, train, predict, parallel, prepost, augment, metrics  # noqa: F401
from .models import UNet3D, AutocastUNet, AutoImplantUNet, DynUNet, SegResNet, UNet, fetch_model_by_name, build_or_load_model  # noqa: F401
from .losses import DiceLoss, DiceCELoss, TverskyLoss, GeneralizedDiceLoss, FocalLoss, DiceFocalLoss  # noqa: F401
from .metrics import HausdorffDistanceMetric, SurfaceDistanceMetric, SurfaceDiceMetric, DiceMetric, MeanIoU, ConfusionMatrixMetric  # noqa: F401,E501
from .predict import SlidingWindowInferer, volumetric_predictions  # noqa: F401
from .train import GraphedTrainStep, epoch_training, batch_loss  # noqa: F401

__version__ = "0.1.0"
