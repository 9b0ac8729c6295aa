"""fadtk_b200 - H100-native drop-in for the embedding -> statistics -> FAD path of microsoft/fadtk.

Export surface mirrors fadtk/__init__.py:1-4 (star re-exports of fad, fad_batch, model_loader,
utils).  Importing the package needs neither a GPU nor the compiled library; the first compute
call loads csrc/libfadtk_b200.so and fails loudly if it or an H100 is missing.
"""
from .fad import *            # noqa: F401,F403
from .fad import FADInfResults, FrechetAudioDistance, calc_embd_statistics, calc_frechet_distance, log  # noqa: F401
from .fad import KADResults, calc_kernel_audio_distance, calc_kernel_audio_distance_songs  # noqa: F401
from .fad import KADComparisonResults, KADTestResults, calc_kad_comparison, calc_kad_test  # noqa: F401
from .fad import FADComparisonResults, calc_fad_comparison  # noqa: F401
from .fad import FADBootstrapResults, KADBootstrapResults, calc_fad_bootstrap, calc_kad_bootstrap  # noqa: F401
from .fad import PRDCResults, calc_prdc, calc_prdc_songs  # noqa: F401
from .fad import RealismResults, calc_realism  # noqa: F401
from .fad import NearestResults, calc_nearest  # noqa: F401
from .fad import prepare_pairwise_baseline  # noqa: F401
from .fad_batch import cache_embedding_files  # noqa: F401
from .layers import cache_layer_embeddings, score_layers  # noqa: F401
from .model_loader import ModelLoader, VGGishModel, CLAPLaionModel, WhisperModel, EncodecEmbModel, Wav2VecFamilyModel, W2V2Model, HuBERTModel, MERTModel, WavLMModel, UnbuiltModel, get_all_models  # noqa: F401
from .utils import (PathLike, DeviceStatistics, calculate_embd_statistics_online,  # noqa: F401
                    find_sox_formats, get_cache_embedding_path, statistics_of_arrays)

__version__ = "0.1.0"
