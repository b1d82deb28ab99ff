"""H100-native (sm_90a) implementation of DAWN's per-step denoising UNet behind the reference's
Python module interface (DynamicNfUnet3D / DynamicNfGaussianDiffusion)."""
from .unet import DynamicNfUnet3D, Unet3D  # noqa: F401
from .diffusion import DynamicNfGaussianDiffusion, GaussianDiffusion  # noqa: F401
from .lfg import Generator as LfgGenerator  # noqa: F401
from .lfg import BGMotionPredictor, FlowAE, MotionGenerator, RegionPredictor  # noqa: F401
from .flow_diffusion import Face_loc_Encoder, FlowDiffusion  # noqa: F401
from .pbnet import get_model as get_pbnet_model  # noqa: F401
from .hubert import HubertModel, hubert_features  # noqa: F401
