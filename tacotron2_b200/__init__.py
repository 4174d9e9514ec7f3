"""tacotron2_b200 -- an H100-native (sm_90a) Tacotron 2 mel-spectrogram engine and WaveGlow vocoder, denoiser
and Griffin-Lim behind the NVIDIA/tacotron2 nn.Module API.  See DESIGN.md / INTEGRATION.md."""
from ._engine import dropout_masks, invalidate_weights  # noqa: F401
from .hparams import create_hparams  # noqa: F401
from .layers import TacotronSTFT  # noqa: F401
from .loss_function import Tacotron2Loss  # noqa: F401
from .model import Decoder, Encoder, Postnet, Tacotron2  # noqa: F401
from . import amp  # noqa: F401
from .glow import WaveGlow, waveglow_noise, window_halo  # noqa: F401
from .denoiser import Denoiser, denoiser_halo  # noqa: F401
from .stft import STFT  # noqa: F401
from .audio_processing import griffin_lim  # noqa: F401
from .optim import AmpFusedClipAdam, FusedClipAdam  # noqa: F401
from .serving import InferenceServer  # noqa: F401

__all__ = ["Tacotron2", "Encoder", "Decoder", "Postnet", "Tacotron2Loss", "create_hparams", "dropout_masks",
           "FusedClipAdam", "AmpFusedClipAdam", "amp", "invalidate_weights", "TacotronSTFT",
           "WaveGlow", "waveglow_noise", "window_halo", "Denoiser", "denoiser_halo", "STFT", "griffin_lim",
           "InferenceServer"]
