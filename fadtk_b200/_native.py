"""ctypes binding of the C ABI in include/fadtk_b200.h (csrc/libfadtk_b200.so).

PyTorch tensors are only containers here: every call passes ``tensor.data_ptr()`` and the
current CUDA stream.  There is no CPU fallback - if the shared library or an H100 is missing
the import of a compute entry point raises.
"""
from __future__ import annotations

import ctypes as C
import json
import os
from pathlib import Path

import numpy as np
import torch

# FADTK_B200_LIB: another build of the same library (A/B measurements of a compile-time variant on one box)
_LIB_PATH = Path(os.environ.get("FADTK_B200_LIB") or Path(__file__).parent / "csrc" / "libfadtk_b200.so")
_lib = None

c_ll = C.c_longlong
c_vp = C.c_void_p


class NativeError(RuntimeError):
    pass


class VggishWeights(C.Structure):
    _fields_ = [("conv1_w_host", c_vp), ("conv1_b_host", c_vp),
                ("conv_w_host", c_vp * 5), ("conv_b_host", c_vp * 5),
                ("fc_w_host", c_vp * 3), ("fc_b_host", c_vp * 3), ("split_mask", C.c_uint32)]


# name -> (restype, argtypes); mirrors include/fadtk_b200.h one to one
SIGNATURES = {
    "fad_version": (C.c_int, []),
    "fad_last_error": (C.c_char_p, []),
    "fad_create": (C.c_int, [C.c_int, C.c_int, C.POINTER(c_vp)]),
    "fad_destroy": (C.c_int, [c_vp]),
    "fad_vggish_load": (C.c_int, [c_vp, C.POINTER(VggishWeights)]),
    "fad_vggish_num_examples": (c_ll, [c_ll]),
    "fad_vggish_plan": (c_ll, [c_vp, c_ll, c_vp, c_ll, c_vp]),
    "fad_vggish_forward": (C.c_int, [c_vp, c_vp, c_vp, c_ll, c_vp, c_vp]),
    "fad_vggish_logmel": (C.c_int, [c_vp, c_vp, c_vp, c_ll, c_vp, C.c_int, c_vp]),
    "fad_vggish_conv1": (C.c_int, [c_vp, c_vp, c_ll, c_vp, c_vp]),
    "fad_umma_layer": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, c_vp,
                                 C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp]),
    "fad_linear": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_ll, c_vp, C.c_int, c_vp, C.c_int, C.c_int, c_vp, c_vp,
                             c_vp, C.c_int, C.c_int, C.c_int, c_vp]),
    "fad_clap_load": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int]),
    "fad_clap_plan": (c_ll, [c_vp, c_ll, c_vp, c_vp, c_ll, c_vp]),
    "fad_clap_plan_frames": (c_ll, [c_vp, c_ll, c_vp, c_vp, c_vp, c_ll, c_vp]),
    "fad_clap_forward": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_ll, c_vp, c_ll, c_vp, c_vp]),
    "fad_clap_logmel": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_ll, c_vp, c_vp]),
    "fad_clap_patch_embed": (C.c_int, [c_vp, c_vp, c_ll, c_vp, c_ll, c_vp, c_vp]),
    "fad_clap_block": (C.c_int, [c_vp, C.c_int, c_vp, c_ll, c_vp, c_vp]),
    "fad_clap_merge": (C.c_int, [c_vp, C.c_int, c_vp, c_ll, c_vp, c_vp]),
    "fad_clap_head": (C.c_int, [c_vp, c_vp, c_ll, c_vp, c_vp]),
    "fad_stats_acc_len": (C.c_size_t, [C.c_int]),
    "fad_stats_accumulate": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, c_vp, C.c_int, c_vp]),
    "fad_stats_accumulate_gather": (C.c_int, [c_vp, c_vp, c_ll, c_vp, c_ll, C.c_int, c_vp, c_vp, c_vp]),
    "fad_stats_finalize": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp]),
    "fad_file_means": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, C.c_int, c_vp, c_vp, c_vp]),
    "fad_stats_accumulate_f64": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, c_vp]),
    "fad_stats_finalize_mirrored": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_int, c_vp, c_vp, c_vp]),
    "fad_frechet": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_sqrt_psd": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, c_vp, c_vp, c_vp]),
    "fad_frechet_presqrt": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_whisper_load": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, C.c_int]),
    "fad_whisper_forward": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_ll, c_vp, c_vp]),
    "fad_whisper_logmel": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_ll, c_vp, c_vp]),
    "fad_whisper_conv": (C.c_int, [c_vp, C.c_int, c_vp, c_vp, c_ll, c_vp, c_vp]),
    "fad_whisper_enc_layer": (C.c_int, [c_vp, C.c_int, c_vp, c_ll, c_vp, c_vp]),
    "fad_whisper_encode": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_ll, c_vp, c_vp]),
    "fad_whisper_dec_layer": (C.c_int, [c_vp, C.c_int, c_vp, c_vp, c_ll, c_vp, c_vp]),
    "fad_w2v_load": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, C.c_int, C.c_int]),
    "fad_w2v_forward": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_w2v_forward_taps": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, C.c_int, c_vp, c_vp]),
    "fad_w2v_normalize": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, c_vp]),
    "fad_w2v_conv": (C.c_int, [c_vp, C.c_int, c_vp, c_ll, C.c_int, c_vp, c_vp]),
    "fad_w2v_posconv": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, c_vp]),
    "fad_w2v_layer": (C.c_int, [c_vp, C.c_int, c_vp, c_ll, C.c_int, c_vp, c_vp]),
    "fad_encodec_load": (C.c_int, [c_vp, c_vp, C.c_int, c_ll, C.c_int]),
    "fad_encodec_forward": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, c_vp]),
    "fad_encodec_conv": (C.c_int, [c_vp, C.c_int, c_vp, c_ll, C.c_int, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_encodec_lstm": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, c_vp]),
    "fad_resample_geometry": (C.c_int, [C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp]),
    "fad_resample_length": (c_ll, [C.c_int, C.c_int, c_ll]),
    "fad_resample_bank": (C.c_int, [C.c_int, C.c_int, c_vp]),
    "fad_resample": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, c_ll, C.c_int, C.c_int, c_vp, c_vp, c_vp]),
    "fad_frechet_batched": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_ll, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_attention": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, C.c_int, c_vp, C.c_int, c_vp]),
    "fad_window_attention": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, C.c_int, c_vp, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_attention_bias": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp]),
    "fad_wavlm_gate": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_ll, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_wavlm_bias_table": (C.c_int, [C.c_int, C.c_int, c_vp, c_vp]),
    "fad_decoder_self_attention": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, c_vp]),
    "fad_cross_attention": (C.c_int, [c_vp, c_vp, c_vp, c_ll, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_layernorm": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_ll, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                c_vp, c_vp, c_vp]),
    "fad_bench_dmma_peak": (C.c_int, [c_vp, C.c_int, c_vp]),
    "fad_kad_median_sq": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, c_vp]),
    "fad_kad_sums": (C.c_int, [c_vp, c_vp, c_ll, c_ll, C.c_int, c_vp, c_vp, c_vp]),
    "fad_kad_song_sums": (C.c_int, [c_vp, c_vp, c_ll, c_vp, c_ll, C.c_int, c_vp, c_vp, c_vp]),
    "fad_kad_median_sq_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, C.c_int, c_vp, c_vp]),
    "fad_kad_sums_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, c_ll, C.c_int, c_vp, c_vp, c_vp]),
    "fad_kad_song_sums_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, c_vp, c_ll, C.c_int, c_vp, c_vp, c_vp]),
    "fad_kad_shard_plan": (C.c_int, [c_vp, c_ll, C.c_int, c_vp]),
    "fad_knn_radii_sq": (C.c_int, [c_vp, c_vp, c_ll, c_ll, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_prdc_counts": (C.c_int, [c_vp, c_vp, c_ll, c_ll, C.c_int, c_vp, c_vp, c_vp, c_vp]),
    "fad_knn_radii_sq_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, c_ll, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_prdc_counts_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, c_ll, C.c_int, c_vp, c_vp, c_vp, c_vp]),
    "fad_knn_song_radii_sq": (C.c_int, [c_vp, c_vp, c_ll, c_vp, c_ll, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_prdc_song_counts": (C.c_int, [c_vp, c_vp, c_ll, c_vp, c_ll, C.c_int, c_vp, c_vp, c_vp, c_vp]),
    "fad_knn_song_radii_sq_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, c_vp, c_ll, C.c_int, C.c_int, c_vp,
                                                c_vp]),
    "fad_prdc_song_counts_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, c_vp, c_ll, C.c_int, c_vp, c_vp, c_vp,
                                               c_vp]),
    "fad_prdc_song_spans": (C.c_int, [c_vp, c_ll, c_ll, c_vp, c_vp]),
    "fad_realism": (C.c_int, [c_vp, c_vp, c_ll, c_ll, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "fad_realism_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, c_ll, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp,
                                      c_vp, c_vp]),
    "fad_nearest": (C.c_int, [c_vp, c_vp, c_ll, c_ll, C.c_int, C.c_int, c_vp, c_ll, c_vp, c_vp, c_vp]),
    "fad_nearest_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, c_ll, C.c_int, C.c_int, c_vp, c_ll, c_vp, c_vp,
                                      c_vp]),
    "fad_pair_digest": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, c_vp]),
    "fad_knn_lists_sq": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_knn_lists_sq_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_kad_eval_sums": (C.c_int, [c_vp, c_vp, c_ll, c_vp, c_ll, C.c_int, c_vp, c_vp, c_vp]),
    "fad_kad_eval_sums_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, c_vp, c_ll, C.c_int, c_vp, c_vp, c_vp]),
    "fad_perm_labels": (C.c_int, [c_vp, c_ll, c_ll, C.c_int, C.c_ulonglong, c_vp, c_vp]),
    "fad_perm_dot": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, c_vp, c_vp]),
    "fad_kad_perm_sums": (C.c_int, [c_vp, c_vp, c_ll, c_ll, C.c_int, c_vp, C.c_int, C.c_ulonglong, c_vp, c_vp]),
    "fad_kad_perm_sums_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, c_ll, C.c_int, c_vp, C.c_int, C.c_ulonglong,
                                            c_vp, c_vp]),
    "fad_record_len": (c_ll, [C.c_int]),
    "fad_unit_records": (C.c_int, [c_vp, c_vp, c_vp, c_ll, C.c_int, c_vp, c_vp, c_vp]),
    "fad_perm_record_sums": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, C.c_int, c_vp, c_vp]),
    "fad_frechet_records": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_ll, C.c_int, c_vp, C.c_int, c_vp, c_vp]),
    "fad_frechet_perm": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_ll, c_ll, C.c_int, C.c_int, C.c_ulonglong,
                                   C.c_int, c_vp, c_vp, c_vp]),
    "fad_boot_counts": (C.c_int, [c_vp, c_ll, C.c_int, C.c_ulonglong, c_vp, c_vp]),
    "fad_boot_record_sums": (C.c_int, [c_vp, c_vp, c_ll, C.c_int, c_vp, C.c_int, c_vp, c_vp]),
    "fad_frechet_boot": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_ll, C.c_int, C.c_int, C.c_ulonglong, C.c_int,
                                   c_vp, c_vp, c_vp]),
    "fad_kad_boot_sums": (C.c_int, [c_vp, c_vp, c_vp, c_ll, C.c_int, c_vp, c_vp, C.c_int, C.c_ulonglong, c_vp, c_vp]),
    "fad_knn_eval_radii_sq": (C.c_int, [c_vp, c_vp, c_ll, c_vp, c_ll, C.c_int, C.c_int, c_vp, c_vp]),
    "fad_knn_eval_radii_sq_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, c_vp, c_ll, C.c_int, C.c_int, c_vp,
                                                c_vp]),
    "fad_realism_prepared": (C.c_int, [c_vp, c_vp, c_ll, c_ll, C.c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "fad_realism_prepared_sharded": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_ll, c_ll, C.c_int, c_vp, c_vp, c_vp, c_vp,
                                               c_vp]),
    "fad_comm_unique_id": (C.c_int, [c_vp]),
    "fad_comm_init": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int]),
    "fad_comm_destroy": (C.c_int, [c_vp]),
    "fad_stats_allreduce": (C.c_int, [c_vp, c_vp, c_vp, C.c_int, c_vp]),
    "fad_allreduce_sum_f64": (C.c_int, [c_vp, c_vp, c_vp, c_ll, c_vp]),
    "fad_launch_count": (c_ll, [c_vp]),
    "fad_profile_enable": (C.c_int, [c_vp, C.c_int]),
    "fad_profile_collect": (C.c_int, [c_vp, c_vp, c_vp, C.c_int]),
}

PROF_CATEGORIES = 20
PROF_NAMES = {0: "logmel", 1: "conv1", 2: "conv2", 3: "conv3_1", 4: "conv3_2", 5: "conv4_1", 6: "conv4_2",
              7: "fc1", 8: "fc2", 9: "fc3", 10: "stats", 11: "stats_reduce", 12: "frechet",
              13: "clap_front", 14: "clap_gemm", 15: "clap_attn", 16: "clap_other"}


def library_path() -> Path:
    return _LIB_PATH


def lib():
    """Load the shared library (built in-tree by ``__graft_entry__.build()``)."""
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise NativeError(
                f"{_LIB_PATH} is missing - run `python -c 'import __graft_entry__ as g; g.build()'`. "
                "fadtk_b200 has no CPU fallback.")
        _lib = C.CDLL(str(_LIB_PATH))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(_lib, name)
            fn.restype = res
            fn.argtypes = args
    return _lib


def _check(rc: int):
    if rc != 0:
        raise NativeError(lib().fad_last_error().decode())


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t) -> int:
    return 0 if t is None else t.data_ptr()


class Engine:
    """One native handle bound to one CUDA device."""

    def __init__(self, device: int | None = None, max_examples: int = 2048):
        if not torch.cuda.is_available():
            raise NativeError("no CUDA device visible: fadtk_b200 has no CPU fallback")
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.max_examples = int(max_examples)
        h = c_vp()
        _check(lib().fad_create(self.device, self.max_examples, C.byref(h)))
        self._h = h
        self._keep = []
        self.has_comm = False     # fad_comm_init done: the statistics all-reduce goes through the C ABI
        self.owners = {}          # weight slot -> token of the loader whose weights it holds (model_loader._DeviceBatch)

    def close(self):
        if getattr(self, "_h", None):
            lib().fad_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def torch_device(self):
        return torch.device("cuda", self.device)

    @property
    def launches(self) -> int:
        return int(lib().fad_launch_count(self._h))

    # ------------------------------------------------------------ cross-GPU merge
    @staticmethod
    def comm_unique_id() -> bytes:
        """rank 0: the 128-byte NCCL rendezvous id (fad_comm_unique_id)"""
        buf = C.create_string_buffer(128)
        _check(lib().fad_comm_unique_id(buf))
        return buf.raw

    def comm_init(self, unique_id: bytes, rank: int, world: int):
        """join the communicator of the C ABI (fad_comm_init); afterwards allreduce_sum_ runs through it"""
        assert len(unique_id) == 128
        _check(lib().fad_comm_init(self._h, C.create_string_buffer(unique_id, 128), int(rank), int(world)))
        self.has_comm = True

    def allreduce_sum_(self, buf: torch.Tensor) -> torch.Tensor:
        """in-place sum of an fp64 cuda tensor over the ranks of the handle's communicator (fad_allreduce_sum_f64)"""
        assert buf.dtype == torch.float64 and buf.is_cuda and buf.is_contiguous()
        _check(lib().fad_allreduce_sum_f64(self._h, None, buf.data_ptr(), buf.numel(), _stream()))
        return buf

    def attention(self, qkv: torch.Tensor, n_clips: int, legacy: bool = False) -> torch.Tensor:
        """qkv fp16 [n_clips * S, 3 d] (cuda) -> fp16 [n_clips * S, d]: per-head softmax(q k^T / 8) v, heads of 64 dims"""
        assert qkv.dtype == torch.float16 and qkv.is_cuda and qkv.is_contiguous() and qkv.shape[0] % n_clips == 0
        S, d = qkv.shape[0] // n_clips, qkv.shape[1] // 3
        out = torch.empty((qkv.shape[0], d), dtype=torch.float16, device=qkv.device)
        _check(lib().fad_attention(self._h, qkv.data_ptr(), n_clips, S, d, out.data_ptr(), int(legacy), _stream()))
        return out

    # Stage entries of the other transformer attention and LayerNorm launches: they write into the caller's cuda
    # tensors (shapes in include/fadtk_b200.h) and raise NativeError on rejected arguments.
    def window_attention(self, qkv, n_windows: int, C: int, heads: int, relbias, res: int, shift: int, out):
        """fad_window_attention: CLAP Swin window attention, qkv fp16 [n_windows * 64, 3 C] -> out fp16 [.., C]"""
        _check(lib().fad_window_attention(self._h, _ptr(qkv), int(n_windows), int(C), int(heads), _ptr(relbias),
                                          int(res), int(shift), _ptr(out), _stream()))
        return out

    def attention_bias(self, qkv, n_clips: int, S: int, d: int, relb, gate, out):
        """fad_attention_bias: WavLM attention with the gated relative position bias, qkv fp16 [n_clips * S, 3 d]"""
        _check(lib().fad_attention_bias(self._h, _ptr(qkv), int(n_clips), int(S), int(d), _ptr(relb), _ptr(gate),
                                        _ptr(out), _stream()))
        return out

    def wavlm_gate(self, x, w, b, c, rows: int, heads: int, d: int, out):
        """fad_wavlm_gate: x fp32 [rows, d] -> out fp32 [rows, heads]"""
        _check(lib().fad_wavlm_gate(self._h, _ptr(x), _ptr(w), _ptr(b), _ptr(c), int(rows), int(heads), int(d),
                                    _ptr(out), _stream()))
        return out

    @staticmethod
    def wavlm_bias_table(rel_embed: np.ndarray, S: int) -> np.ndarray:
        """rel_embed float32 [320, heads] -> float32 [heads, 2 S - 1], the table fad_w2v_forward uploads (host only)"""
        emb = np.ascontiguousarray(rel_embed, dtype=np.float32)
        out = np.empty((emb.shape[1], max(2 * int(S) - 1, 0)), dtype=np.float32)
        _check(lib().fad_wavlm_bias_table(emb.shape[1], int(S), emb.ctypes.data, out.ctypes.data))
        return out

    def decoder_self_attention(self, qkv, n_clips: int, d: int, out):
        """fad_decoder_self_attention: Whisper decoder, qkv fp16 [n_clips * 2, 3 d] -> out fp16 [n_clips * 2, d]"""
        _check(lib().fad_decoder_self_attention(self._h, _ptr(qkv), int(n_clips), int(d), _ptr(out), _stream()))
        return out

    def cross_attention(self, q, kv, n_clips: int, S: int, d: int, out):
        """fad_cross_attention: q fp16 [n_clips * 2, d], kv fp16 [n_clips * S, 2 d] -> out fp16 [n_clips * 2, d]"""
        _check(lib().fad_cross_attention(self._h, _ptr(q), _ptr(kv), int(n_clips), int(S), int(d), _ptr(out), _stream()))
        return out

    def layernorm(self, x, gamma, beta, rows: int, C: int, ld_out: int, out16, out32=None, *, res: int = 0,
                  shift: int = 0, mode: int = 0, gelu: bool = False):
        """fad_layernorm: x fp32 -> out16 fp16 [rows, ld_out] (and out32 fp32 [rows, width] if given)"""
        _check(lib().fad_layernorm(self._h, _ptr(x), _ptr(gamma), _ptr(beta), int(rows), int(C), int(ld_out), int(res),
                                   int(shift), int(mode), int(gelu), _ptr(out16), _ptr(out32), _stream()))
        return out16

    def dmma_peak_tflops(self, iters: int = 0) -> float:
        """measured fp64 tensor-pipe (DMMA) rate, TFLOP/s: roofline denominator of the fp64 kernels"""
        out = C.c_double(0.0)
        _check(lib().fad_bench_dmma_peak(self._h, int(iters), C.byref(out)))
        return float(out.value)

    def profile(self, on: bool):
        _check(lib().fad_profile_enable(self._h, int(on)))

    def profile_collect(self, reset: bool = True) -> dict:
        """-> {category: (milliseconds, launches)} measured with CUDA events on the launch stream."""
        ms = (C.c_double * PROF_CATEGORIES)()
        cnt = (c_ll * PROF_CATEGORIES)()
        _check(lib().fad_profile_collect(self._h, ms, cnt, int(reset)))
        return {PROF_NAMES[i]: (ms[i], int(cnt[i])) for i in PROF_NAMES if cnt[i]}

    # ------------------------------------------------------------------ VGGish
    def vggish_load(self, packed: dict):
        """``packed`` comes from fadtk_b200.weights.pack_vggish (CPU tensors)."""
        self.owners.pop("vggish", None)          # whoever loads claims the slot afterwards (model_loader._DeviceBatch)
        w = VggishWeights()
        keep = {k: v.contiguous() for k, v in packed.items() if hasattr(v, "contiguous")}
        w.conv1_w_host = keep["conv1.w"].data_ptr()
        w.conv1_b_host = keep["conv1.b"].data_ptr()
        for i in range(5):
            w.conv_w_host[i] = keep[f"conv{i + 2}.w"].data_ptr()
            w.conv_b_host[i] = keep[f"conv{i + 2}.b"].data_ptr()
        for i in range(3):
            w.fc_w_host[i] = keep[f"fc{i + 1}.w"].data_ptr()
            w.fc_b_host[i] = keep[f"fc{i + 1}.b"].data_ptr()
        w.split_mask = int(packed.get("split_mask", 0))
        _check(lib().fad_vggish_load(self._h, C.byref(w)))

    @staticmethod
    def vggish_plan(clip_offsets: np.ndarray):
        """-> (ex_start int64 [n_examples], rows_per_clip int64 [n_clips])"""
        off = np.ascontiguousarray(clip_offsets, dtype=np.int64)
        n_clips = off.shape[0] - 1
        rows = np.empty(n_clips, dtype=np.int64)
        n = lib().fad_vggish_plan(off.ctypes.data, n_clips, None, 0, rows.ctypes.data)
        ex = np.empty(n, dtype=np.int64)
        lib().fad_vggish_plan(off.ctypes.data, n_clips, ex.ctypes.data, n, None)
        return ex, rows

    def vggish_forward(self, pcm: torch.Tensor, ex_start: torch.Tensor, out: torch.Tensor | None = None):
        """pcm int16 [samples] (cuda), ex_start int64 [n] (cuda) -> fp16 [n, 128] (cuda)."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda and pcm.is_contiguous()
        assert ex_start.dtype == torch.int64 and ex_start.is_cuda
        n = ex_start.shape[0]
        if out is None:
            out = torch.empty((n, 128), dtype=torch.float16, device=pcm.device)
        assert out.dtype == torch.float16 and out.is_contiguous() and out.shape[0] >= n
        _check(lib().fad_vggish_forward(self._h, pcm.data_ptr(), ex_start.data_ptr(), n,
                                        out.data_ptr(), _stream()))
        return out[:n]

    def vggish_logmel(self, pcm, ex_start, use_double=True):
        n = ex_start.shape[0]
        out = torch.empty((n, 96, 64), dtype=torch.float32, device=pcm.device)
        _check(lib().fad_vggish_logmel(self._h, pcm.data_ptr(), ex_start.data_ptr(), n,
                                       out.data_ptr(), int(use_double), _stream()))
        return out

    def vggish_conv1(self, logmel):
        """fp32 [n, 96, 64] log-mel examples -> fp16 NHWC [n, 48, 32, 64] (conv1 + ReLU + max-pool, loaded weights)"""
        assert logmel.dtype == torch.float32 and logmel.is_contiguous() and logmel.shape[1:] == (96, 64)
        n = logmel.shape[0]
        out = torch.empty((n, 48, 32, 64), dtype=torch.float16, device=logmel.device)
        _check(lib().fad_vggish_conv1(self._h, logmel.data_ptr(), n, out.data_ptr(), _stream()))
        return out

    def umma_layer(self, x, w, bias, taps, relu, pool, want_f32=False, split_w=False):
        """x fp16 NHWC [NB,H,W,Cin]; w fp16 [Cout, taps*Cin] (or [2*Cout, taps*Cin] hi/lo tiles when
        split_w, see weights.split_hi_lo_tiles); bias fp32 [Cout]."""
        nb, hh, ww, cin = x.shape
        cout = w.shape[0] // (2 if split_w else 1)
        oh, ow = (hh // 2, ww // 2) if pool else (hh, ww)
        out = torch.empty((nb, oh, ow, cout), dtype=torch.float16, device=x.device)
        out32 = torch.empty((nb, oh, ow, cout), dtype=torch.float32, device=x.device) if want_f32 else None
        _check(lib().fad_umma_layer(self._h, x.data_ptr(), nb, hh, ww, cin, w.data_ptr(), bias.data_ptr(),
                                    cout, taps, int(relu), int(pool), int(split_w), out.data_ptr(), _ptr(out32),
                                    _stream()))
        return (out, out32) if want_f32 else out

    def linear(self, a, rows: int, k_cols: int, w, bias, n_cols: int, act: int = 0, *, lda: int = 0, split_w: int = 1,
               out16=None, out32=None, resid=None, resid_C: int = 0, resid_res: int = 0, resid_shift: int = 0):
        """fad_linear: act(A W^T + bias) into the caller's buffers (cuda tensors, any of out16 / out32 / resid).
        a fp16 rows of k_cols elements lda apart (0: k_cols); w packed fp16 [(2 if split_w else 1) * pad128(n_cols),
        pad64(k_cols)]; bias fp32 [pad128(n_cols)]; out16 / out32 [rows, n_cols] from their first element;
        resid fp32 [tokens, resid_C] updated in place.  Raises NativeError on rejected arguments."""
        _check(lib().fad_linear(self._h, _ptr(a), int(rows), int(k_cols), int(lda), _ptr(w), int(split_w),
                                _ptr(bias), int(n_cols), int(act), _ptr(out16), _ptr(out32), _ptr(resid),
                                int(resid_C), int(resid_res), int(resid_shift), _stream()))

    # -------------------------------------------------------------------- CLAP
    def clap_load(self, tensors: list, max_chunks: int = 32):
        """``tensors`` comes from fadtk_b200.weights_clap.pack_clap (CPU tensors, fixed order)."""
        self.owners.pop("clap", None)          # whoever loads claims the slot afterwards (model_loader._DeviceBatch)
        keep = [t.contiguous() for t in tensors]
        arr = (c_vp * len(keep))(*[t.data_ptr() for t in keep])
        _check(lib().fad_clap_load(self._h, arr, len(keep), int(max_chunks)))

    @staticmethod
    def clap_plan(clip_offsets: np.ndarray):
        """-> (chunk_start int64 [n], chunk_valid int32 [n], rows_per_clip int64 [n_clips])"""
        off = np.ascontiguousarray(clip_offsets, dtype=np.int64)
        n_clips = off.shape[0] - 1
        rows = np.empty(n_clips, dtype=np.int64)
        n = lib().fad_clap_plan(off.ctypes.data, n_clips, None, None, 0, rows.ctypes.data)
        start = np.empty(n, dtype=np.int64)
        valid = np.empty(n, dtype=np.int32)
        lib().fad_clap_plan(off.ctypes.data, n_clips, start.ctypes.data, valid.ctypes.data, n, None)
        return start, valid, rows

    @staticmethod
    def clap_plan_frames(clip_offsets: np.ndarray):
        """-> dict(pool_start int64, pool_valid int32, pool_frame int32, frame_index int32 [n_chunks,1001],
        rows_per_clip int64): every distinct STFT frame once + the per-window index table."""
        off = np.ascontiguousarray(clip_offsets, dtype=np.int64)
        n_clips = off.shape[0] - 1
        rows = np.empty(n_clips, dtype=np.int64)
        n_chunks = lib().fad_clap_plan(off.ctypes.data, n_clips, None, None, 0, rows.ctypes.data)
        n_pool = lib().fad_clap_plan_frames(off.ctypes.data, n_clips, None, None, None, 0, None)
        ps = np.empty(n_pool, dtype=np.int64)
        pv = np.empty(n_pool, dtype=np.int32)
        pf = np.empty(n_pool, dtype=np.int32)
        fi = np.empty((n_chunks, 1001), dtype=np.int32)
        lib().fad_clap_plan_frames(off.ctypes.data, n_clips, ps.ctypes.data, pv.ctypes.data, pf.ctypes.data, n_pool,
                                   fi.ctypes.data)
        return {"pool_start": ps, "pool_valid": pv, "pool_frame": pf, "frame_index": fi, "rows_per_clip": rows}

    def clap_plan_to_device(self, plan: dict) -> dict:
        dev = self.torch_device
        return {k: (torch.from_numpy(v).to(dev) if k != "rows_per_clip" else v) for k, v in plan.items()}

    def clap_forward(self, pcm: torch.Tensor, plan_dev: dict):
        """pcm int16 (cuda, 48 kHz); plan_dev from clap_plan_to_device -> fp16 [n_chunks, 512]."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda
        fi = plan_dev["frame_index"]
        n = fi.shape[0]
        out = torch.empty((n, 512), dtype=torch.float16, device=pcm.device)
        _check(lib().fad_clap_forward(self._h, pcm.data_ptr(), plan_dev["pool_start"].data_ptr(),
                                      plan_dev["pool_valid"].data_ptr(), plan_dev["pool_frame"].data_ptr(),
                                      plan_dev["pool_start"].shape[0], fi.data_ptr(), n, out.data_ptr(), _stream()))
        return out

    def clap_logmel(self, pcm, plan_dev: dict):
        """-> fp32 [n_chunks, 1001, 64] BatchNorm-ed log-mel, gathered from the frame pool."""
        n_pool = plan_dev["pool_start"].shape[0]
        pool = torch.empty((n_pool, 64), dtype=torch.float32, device=pcm.device)
        _check(lib().fad_clap_logmel(self._h, pcm.data_ptr(), plan_dev["pool_start"].data_ptr(),
                                     plan_dev["pool_valid"].data_ptr(), plan_dev["pool_frame"].data_ptr(), n_pool,
                                     pool.data_ptr(), _stream()))
        return pool[plan_dev["frame_index"].long()]

    # Stage entries of the loaded CLAP model: they write into the caller's cuda tensors (shapes in
    # include/fadtk_b200.h) and raise NativeError on rejected arguments.
    def clap_pool(self, pcm, pool_start, pool_valid, pool_frame, n_pool: int, out):
        """fad_clap_logmel: out fp32 [n_pool, 64], the BatchNorm-ed log-mel row of every frame-pool entry"""
        _check(lib().fad_clap_logmel(self._h, _ptr(pcm), _ptr(pool_start), _ptr(pool_valid), _ptr(pool_frame),
                                     int(n_pool), _ptr(out), _stream()))
        return out

    def clap_patch_embed(self, pool, n_pool: int, frame_index, B: int, out):
        """fad_clap_patch_embed: pool fp32 [n_pool, 64], frame_index int32 [B, 1001] -> out fp32 [B, 4096, E]"""
        _check(lib().fad_clap_patch_embed(self._h, _ptr(pool), int(n_pool), _ptr(frame_index), int(B), _ptr(out),
                                          _stream()))
        return out

    def clap_block(self, blk: int, x, B: int, out):
        """fad_clap_block: Swin block blk, x fp32 [B, res^2, C] -> out fp32 [B, res^2, C]"""
        _check(lib().fad_clap_block(self._h, int(blk), _ptr(x), int(B), _ptr(out), _stream()))
        return out

    def clap_merge(self, s: int, x, B: int, out):
        """fad_clap_merge: patch merge s, x fp32 [B, res^2, C] -> out fp32 [B, res^2 / 4, 2 C]"""
        _check(lib().fad_clap_merge(self._h, int(s), _ptr(x), int(B), _ptr(out), _stream()))
        return out

    def clap_head(self, x, B: int, out):
        """fad_clap_head: x fp32 [B, 64, 8 E] -> out fp16 [B, 512]"""
        _check(lib().fad_clap_head(self._h, _ptr(x), int(B), _ptr(out), _stream()))
        return out

    def clap_forward_raw(self, pcm, pool_start, pool_valid, pool_frame, n_pool: int, frame_index, n_chunks: int, out):
        """fad_clap_forward with every pointer and count as given (None -> NULL)"""
        _check(lib().fad_clap_forward(self._h, _ptr(pcm), _ptr(pool_start), _ptr(pool_valid), _ptr(pool_frame),
                                      int(n_pool), _ptr(frame_index), int(n_chunks), _ptr(out), _stream()))
        return out

    # ------------------------------------------------------------------ Whisper
    def whisper_load(self, cfg: tuple, tensors: list, max_clips: int = 16):
        """cfg = (d_model, heads, enc_layers, dec_layers, ffn); tensors from weights_whisper.pack_whisper."""
        self.owners.pop("whisper", None)          # whoever loads claims the slot afterwards (model_loader._DeviceBatch)
        keep = [t.contiguous() for t in tensors]
        arr = (c_vp * len(keep))(*[t.data_ptr() for t in keep])
        c = (C.c_int * 5)(*[int(v) for v in cfg])
        _check(lib().fad_whisper_load(self._h, c, arr, len(keep), int(max_clips)))
        self._whisper_d = int(cfg[0])

    def whisper_forward(self, pcm: torch.Tensor, clip_start: torch.Tensor, clip_len: torch.Tensor) -> torch.Tensor:
        """pcm int16 (cuda, 16 kHz); clip_start int64 / clip_len int32 [n] (cuda) -> fp16 [n, 2, d_model]."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda and clip_start.dtype == torch.int64 and clip_len.dtype == torch.int32
        n = clip_start.shape[0]
        out = torch.empty((n, 2, self._whisper_d), dtype=torch.float16, device=pcm.device)
        _check(lib().fad_whisper_forward(self._h, pcm.data_ptr(), clip_start.data_ptr(), clip_len.data_ptr(), n,
                                         out.data_ptr(), _stream()))
        return out

    def whisper_features(self, pcm: torch.Tensor, clip_start: torch.Tensor, clip_len: torch.Tensor) -> torch.Tensor:
        """-> fp32 [n, 3000, 80]: the feature extractor's input_features (time-major)."""
        n = clip_start.shape[0]
        buf = torch.empty(n * 3000 * 80 + n, dtype=torch.float32, device=pcm.device)
        _check(lib().fad_whisper_logmel(self._h, pcm.data_ptr(), clip_start.data_ptr(), clip_len.data_ptr(), n,
                                        buf.data_ptr(), _stream()))
        raw = buf[: n * 3000 * 80].view(n, 3000, 80)
        mx = buf[n * 3000 * 80:].view(n, 1, 1)
        return (torch.maximum(raw, mx - 8.0) + 4.0) / 4.0

    # Stage entries of the loaded Whisper model: they write into the caller's cuda tensors (shapes in
    # include/fadtk_b200.h) and raise NativeError on rejected arguments.
    def whisper_logmel(self, pcm, clip_start, clip_len, n_clips: int, out):
        """fad_whisper_logmel: out fp32 [n_clips * 3000 * 80 + n_clips], the raw log10 mel then the per-clip maxima"""
        _check(lib().fad_whisper_logmel(self._h, _ptr(pcm), _ptr(clip_start), _ptr(clip_len), int(n_clips), _ptr(out),
                                        _stream()))
        return out

    def whisper_conv(self, c: int, x, clip_max, B: int, out):
        """fad_whisper_conv: c = 0 raw log10 mel fp32 [B, 3000, 80] + clip_max fp32 [B] -> out fp16 [B, 3000, d];
        c = 1 fp16 [B, 3000, d] -> out fp32 [B, 1500, d]"""
        _check(lib().fad_whisper_conv(self._h, int(c), _ptr(x), _ptr(clip_max), int(B), _ptr(out), _stream()))
        return out

    def whisper_enc_layer(self, l: int, x, B: int, out):
        """fad_whisper_enc_layer: encoder layer l, x fp32 [B, 1500, d] -> out fp32 [B, 1500, d]"""
        _check(lib().fad_whisper_enc_layer(self._h, int(l), _ptr(x), int(B), _ptr(out), _stream()))
        return out

    def whisper_encode(self, pcm, clip_start, clip_len, n_clips: int, out):
        """fad_whisper_encode: the encoder with its final LayerNorm -> out fp16 [n_clips, 1500, d]"""
        _check(lib().fad_whisper_encode(self._h, _ptr(pcm), _ptr(clip_start), _ptr(clip_len), int(n_clips), _ptr(out),
                                        _stream()))
        return out

    def whisper_dec_layer(self, l: int, xd, enc_out, B: int, out):
        """fad_whisper_dec_layer: decoder layer l, xd fp32 [B, 2, d], enc_out fp16 [B, 1500, d] -> out fp32 [B, 2, d]"""
        _check(lib().fad_whisper_dec_layer(self._h, int(l), _ptr(xd), _ptr(enc_out), int(B), _ptr(out), _stream()))
        return out

    # ------------------------------------------------------- wav2vec 2.0 / HuBERT / MERT
    def w2v_load(self, cfg: tuple, tensors: list, max_clips: int = 8, max_len: int = 16000 * 30):
        """cfg = weights_w2v.config_of(state); tensors from weights_w2v.pack_w2v."""
        self.owners.pop("w2v", None)          # whoever loads claims the slot afterwards (model_loader._DeviceBatch)
        keep = [t.contiguous() for t in tensors]
        arr = (c_vp * len(keep))(*[t.data_ptr() for t in keep])
        c = (C.c_int * 7)(*[int(v) for v in cfg])
        _check(lib().fad_w2v_load(self._h, c, arr, len(keep), int(max_clips), int(max_len)))
        self._w2v_d = int(cfg[0])

    @staticmethod
    def w2v_frames(n_samples: int) -> int:
        t = n_samples
        for k, s in zip((10, 3, 3, 3, 3, 2, 2), (5, 2, 2, 2, 2, 2, 2)):
            t = (t - k) // s + 1
        return t

    def w2v_forward(self, pcm: torch.Tensor, layer: int) -> torch.Tensor:
        """pcm int16 [n_clips, L] (cuda, equal lengths) -> fp16 [n_clips, frames, d_model] = hidden_states[layer]."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda and pcm.ndim == 2 and pcm.is_contiguous()
        n, L = pcm.shape
        out = torch.empty((n, self.w2v_frames(L), self._w2v_d), dtype=torch.float16, device=pcm.device)
        _check(lib().fad_w2v_forward(self._h, pcm.data_ptr(), n, L, int(layer), out.data_ptr(), _stream()))
        return out

    def w2v_forward_taps(self, pcm: torch.Tensor, taps, out=None) -> torch.Tensor:
        """pcm int16 [n_clips, L] (cuda, equal lengths), taps strictly increasing layers -> fp16
        [n_taps, n_clips, frames, d_model], slice t = hidden_states[taps[t]] from ONE forward (written into `out` when
        given)."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda and pcm.ndim == 2 and pcm.is_contiguous()
        n, L = pcm.shape
        taps = [int(t) for t in taps]
        if out is None:
            out = torch.empty((len(taps), n, self.w2v_frames(L), self._w2v_d), dtype=torch.float16, device=pcm.device)
        arr = (C.c_int * max(1, len(taps)))(*taps)
        _check(lib().fad_w2v_forward_taps(self._h, pcm.data_ptr(), n, L, arr, len(taps), _ptr(out), _stream()))
        return out

    # Stage entries of the loaded encoder: they write into the caller's cuda tensors (shapes in include/fadtk_b200.h)
    # and raise NativeError on rejected arguments.
    def w2v_normalize(self, pcm, n_clips: int, L: int, out):
        """fad_w2v_normalize: pcm int16 [n_clips, L] -> out fp32 [n_clips, L]"""
        _check(lib().fad_w2v_normalize(self._h, _ptr(pcm), int(n_clips), int(L), _ptr(out), _stream()))
        return out

    def w2v_conv(self, c: int, x, B: int, L: int, out):
        """fad_w2v_conv: feature-encoder conv c at the frames of L-sample clips; x [B, T_c, 512] (c = 0: fp32 [B, L])
        -> out [B, T_c+1, 512] (fp16; c = 6: fp32)"""
        _check(lib().fad_w2v_conv(self._h, int(c), _ptr(x), int(B), int(L), _ptr(out), _stream()))
        return out

    def w2v_posconv(self, x, B: int, S: int, out):
        """fad_w2v_posconv: x fp32 [B, S, d] -> out fp32 [B, S, d] = x + GELU(pos_conv(x))"""
        _check(lib().fad_w2v_posconv(self._h, _ptr(x), int(B), int(S), _ptr(out), _stream()))
        return out

    def w2v_layer(self, l: int, x, B: int, S: int, out):
        """fad_w2v_layer: encoder layer l, x fp32 [B, S, d] (the stream entering it) -> out fp32 [B, S, d]"""
        _check(lib().fad_w2v_layer(self._h, int(l), _ptr(x), int(B), int(S), _ptr(out), _stream()))
        return out

    # ------------------------------------------------------------------ Encodec
    def encodec_load(self, tensors: list, max_chunk_samples: int = 16 * 240000, variant: str = "24k"):
        self.owners.pop("encodec", None)          # whoever loads claims the slot afterwards (model_loader._DeviceBatch)
        keep = [t.contiguous() for t in tensors]
        arr = (c_vp * len(keep))(*[t.data_ptr() for t in keep])
        _check(lib().fad_encodec_load(self._h, arr, len(keep), int(max_chunk_samples), 0 if variant == "24k" else 1))

    def encodec_forward(self, pcm: torch.Tensor) -> torch.Tensor:
        """pcm int16 [n_clips, T] (cuda, 24 kHz, equal lengths) -> fp16 [n_clips, ceil(T/320), 128]."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda and pcm.ndim == 2 and pcm.is_contiguous()
        n, T = pcm.shape
        frames = T
        for r in (2, 4, 5, 8):
            frames = -(-frames // r)
        out = torch.empty((n, frames, 128), dtype=torch.float16, device=pcm.device)
        _check(lib().fad_encodec_forward(self._h, pcm.data_ptr(), n, T, out.data_ptr(), _stream()))
        return out

    # Stage entries of the loaded encoder: they write into the caller's cuda tensors (shapes in include/fadtk_b200.h)
    # and raise NativeError on rejected arguments.
    def encodec_conv(self, layer: int, x, B: int, T_in: int, out, *, elu_in: bool = False, groupnorm: bool = False):
        """fad_encodec_conv: conv `layer` (load order), x fp32 [B, T_in, Cin] -> out fp32 [B, ceil(T_in / stride), Cout]"""
        _check(lib().fad_encodec_conv(self._h, int(layer), _ptr(x), int(B), int(T_in), int(elu_in), int(groupnorm),
                                      _ptr(out), _stream()))
        return out

    def encodec_lstm(self, z, n_clips: int, TF: int, out):
        """fad_encodec_lstm: z fp32 [n_clips, TF, 512] -> out fp32 [n_clips, TF, 512] = LSTM(z) + z"""
        _check(lib().fad_encodec_lstm(self._h, _ptr(z), int(n_clips), int(TF), _ptr(out), _stream()))
        return out

    # -------------------------------------------------------------- audio conversion
    @staticmethod
    def resample_geometry(sr_in: int, sr_out: int):
        """-> (orig, new, width, taps) of torchaudio's polyphase resampler for this rate pair."""
        v = [C.c_int() for _ in range(4)]
        _check(lib().fad_resample_geometry(int(sr_in), int(sr_out), *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    @staticmethod
    def resample_bank(sr_in: int, sr_out: int) -> np.ndarray:
        """float32 [new, taps] filter bank (host only; what fad_resample uploads)."""
        _, new, _, taps = Engine.resample_geometry(sr_in, sr_out)
        bank = np.empty((new, taps), dtype=np.float32)
        _check(lib().fad_resample_bank(int(sr_in), int(sr_out), bank.ctypes.data))
        return bank

    def resample(self, x: torch.Tensor, sr_in: int, sr_out: int, return_float: bool = False):
        """x: int16 [length, channels] / [length] (PCM16, cuda) or float32 [channels, length] (cuda)
        -> int16 [ceil(new*length/orig)] mono at sr_out (and the un-quantised float32 if asked)."""
        assert x.is_cuda
        if x.dtype == torch.int16:
            x = x.contiguous()
            length, channels = x.shape[0], (1 if x.ndim == 1 else x.shape[1])
            pi, pf = x.data_ptr(), None
        else:
            assert x.dtype == torch.float32 and x.ndim == 2
            x = x.contiguous()
            channels, length = x.shape
            pi, pf = None, x.data_ptr()
        n_out = int(lib().fad_resample_length(int(sr_in), int(sr_out), length))
        out = torch.empty(n_out, dtype=torch.int16, device=x.device)
        outf = torch.empty(n_out, dtype=torch.float32, device=x.device) if return_float else None
        _check(lib().fad_resample(self._h, pi, pf, channels, length, int(sr_in), int(sr_out), out.data_ptr(),
                                  outf.data_ptr() if outf is not None else None, _stream()))
        return (out, outf) if return_float else out

    # -------------------------------------------------------------- statistics
    @staticmethod
    def stats_acc_len(d: int) -> int:
        return int(lib().fad_stats_acc_len(d))

    def stats_new(self, d: int) -> torch.Tensor:
        return torch.zeros(self.stats_acc_len(d), dtype=torch.float64, device=self.torch_device)

    def stats_accumulate(self, emb, shift, acc, tensor_core: int = 0):
        """tensor_core 0: exact Gram on the FP64 tensor pipe (the product path); 2: the CUDA-core fp64 cross-check."""
        assert emb.dtype == torch.float16 and emb.is_contiguous() and shift.dtype == torch.float16
        n, d = emb.shape
        _check(lib().fad_stats_accumulate(self._h, emb.data_ptr(), n, d, shift.data_ptr(),
                                          acc.data_ptr(), int(tensor_core), _stream()))
        return acc

    def stats_accumulate_gather(self, emb, idx, shift, acc):
        assert emb.dtype == torch.float16 and emb.is_contiguous() and idx.dtype == torch.int64
        n, d = emb.shape
        _check(lib().fad_stats_accumulate_gather(self._h, emb.data_ptr(), n, idx.data_ptr(), idx.shape[0], d,
                                                 shift.data_ptr(), acc.data_ptr(), _stream()))
        return acc

    def stats_finalize(self, acc, shift, d):
        mu = torch.empty(d, dtype=torch.float64, device=acc.device)
        cov = torch.empty((d, d), dtype=torch.float64, device=acc.device)
        _check(lib().fad_stats_finalize(self._h, acc.data_ptr(), shift.data_ptr(), d,
                                        mu.data_ptr(), cov.data_ptr(), _stream()))
        return mu, cov

    def file_means(self, emb: torch.Tensor, rows_per_file: int):
        """fp16 [n_files * r, d] -> (m64, m16) fp64 [n_files, d]: exact per-file means and the reference's fp16-rounded ones"""
        n_files, d = emb.shape[0] // rows_per_file, emb.shape[1]
        m64 = torch.empty((n_files, d), dtype=torch.float64, device=emb.device)
        m16 = torch.empty_like(m64)
        _check(lib().fad_file_means(self._h, emb.data_ptr(), n_files, rows_per_file, d, m64.data_ptr(), m16.data_ptr(), _stream()))
        return m64, m16

    def stats_accumulate_f64(self, rows: torch.Tensor, acc: torch.Tensor) -> torch.Tensor:
        assert rows.dtype == torch.float64 and rows.is_contiguous()
        _check(lib().fad_stats_accumulate_f64(self._h, rows.data_ptr(), rows.shape[0], rows.shape[1], acc.data_ptr(), _stream()))
        return acc

    def stats_finalize_mirrored(self, acc, acc64, acc16, shift, rows_per_file: int, d: int):
        """(mu, cov) as the reference's calculate_embd_statistics_online gives them for equal-length files (utils.py:13-46)"""
        mu = torch.empty(d, dtype=torch.float64, device=acc.device)
        cov = torch.empty((d, d), dtype=torch.float64, device=acc.device)
        _check(lib().fad_stats_finalize_mirrored(self._h, acc.data_ptr(), acc64.data_ptr(), acc16.data_ptr(), shift.data_ptr(),
                                                 int(rows_per_file), d, mu.data_ptr(), cov.data_ptr(), _stream()))
        return mu, cov

    # ----------------------------------------------------------------- Frechet
    def frechet(self, mu1, cov1, mu2, cov2, iters: int = 0) -> torch.Tensor:
        """fp64 cuda tensors -> fp64 [8] cuda: FAD, tr sqrt, residual, iters, |dmu|^2, trC1, trC2."""
        d = mu1.shape[0]
        for t in (mu1, cov1, mu2, cov2):
            assert t.dtype == torch.float64 and t.is_cuda and t.is_contiguous()
        out = torch.zeros(8, dtype=torch.float64, device=mu1.device)
        _check(lib().fad_frechet(self._h, mu1.data_ptr(), cov1.data_ptr(), mu2.data_ptr(), cov2.data_ptr(),
                                 d, iters, out.data_ptr(), _stream()))
        return out

    # --------------------------------------------------------- Kernel Audio Distance
    def kad_median_sq(self, x: torch.Tensor) -> torch.Tensor:
        """x fp16 [m, d] (cuda, d a multiple of 8) -> fp64 [2] (cuda): the two middle squared distances of the pairs
        i < j of x (fad_kad_median_sq; equal when m (m - 1) / 2 is odd)."""
        assert x.dtype == torch.float16 and x.is_cuda and x.is_contiguous() and x.ndim == 2
        out = torch.empty(2, dtype=torch.float64, device=x.device)
        _check(lib().fad_kad_median_sq(self._h, x.data_ptr(), x.shape[0], x.shape[1], out.data_ptr(), _stream()))
        return out

    def kad_sums(self, z: torch.Tensor, m: int, sigma: torch.Tensor) -> torch.Tensor:
        """z fp16 [m + n, d] (cuda, X rows first), sigma fp64 scalar (cuda) -> fp64 [3] (cuda): S_xx, S_yy (pairs i < j)
        and S_xy of exp(-|a - b|^2 / (2 sigma^2)) (fad_kad_sums)."""
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        assert sigma.dtype == torch.float64 and sigma.is_cuda and sigma.numel() == 1
        out = torch.empty(3, dtype=torch.float64, device=z.device)
        _check(lib().fad_kad_sums(self._h, z.data_ptr(), int(m), z.shape[0] - int(m), z.shape[1], sigma.data_ptr(),
                                  out.data_ptr(), _stream()))
        return out

    def kad_song_sums(self, z: torch.Tensor, m: int, offsets: torch.Tensor, sigma: torch.Tensor) -> torch.Tensor:
        """z fp16 [m + n_total, d] (cuda, X rows first), offsets int64 [n_items + 1] (cuda, into the rows after X),
        sigma fp64 scalar (cuda) -> fp64 [1 + 2 n_items] (cuda): S_xx, then S_yy,k and S_xy,k per song
        (fad_kad_song_sums)."""
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous() and offsets.ndim == 1
        assert sigma.dtype == torch.float64 and sigma.is_cuda and sigma.numel() == 1
        n_items = offsets.shape[0] - 1
        out = torch.empty(1 + 2 * n_items, dtype=torch.float64, device=z.device)
        _check(lib().fad_kad_song_sums(self._h, z.data_ptr(), int(m), offsets.data_ptr(), n_items, z.shape[1],
                                       sigma.data_ptr(), out.data_ptr(), _stream()))
        return out

    # The same three results with the tile work split into shards (include/fadtk_b200.h): local_shards = 0 is
    # collective over the handle's communicator (comm_init), every rank getting the whole output; local_shards >= 1
    # runs that many shards one after another on this device.  Outputs are bitwise equal to the unsharded entries.
    def kad_median_sq_sharded(self, x: torch.Tensor, local_shards: int = 0) -> torch.Tensor:
        """fad_kad_median_sq_sharded: kad_median_sq over shards"""
        assert x.dtype == torch.float16 and x.is_cuda and x.is_contiguous() and x.ndim == 2
        out = torch.empty(2, dtype=torch.float64, device=x.device)
        _check(lib().fad_kad_median_sq_sharded(self._h, None, int(local_shards), x.data_ptr(), x.shape[0], x.shape[1],
                                               out.data_ptr(), _stream()))
        return out

    def kad_sums_sharded(self, z: torch.Tensor, m: int, sigma: torch.Tensor, local_shards: int = 0) -> torch.Tensor:
        """fad_kad_sums_sharded: kad_sums over shards"""
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        assert sigma.dtype == torch.float64 and sigma.is_cuda and sigma.numel() == 1
        out = torch.empty(3, dtype=torch.float64, device=z.device)
        _check(lib().fad_kad_sums_sharded(self._h, None, int(local_shards), z.data_ptr(), int(m), z.shape[0] - int(m),
                                          z.shape[1], sigma.data_ptr(), out.data_ptr(), _stream()))
        return out

    def kad_song_sums_sharded(self, z: torch.Tensor, m: int, offsets: torch.Tensor, sigma: torch.Tensor,
                              local_shards: int = 0) -> torch.Tensor:
        """fad_kad_song_sums_sharded: kad_song_sums over shards"""
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous() and offsets.ndim == 1
        assert sigma.dtype == torch.float64 and sigma.is_cuda and sigma.numel() == 1
        n_items = offsets.shape[0] - 1
        out = torch.empty(1 + 2 * n_items, dtype=torch.float64, device=z.device)
        _check(lib().fad_kad_song_sums_sharded(self._h, None, int(local_shards), z.data_ptr(), int(m), offsets.data_ptr(),
                                               n_items, z.shape[1], sigma.data_ptr(), out.data_ptr(), _stream()))
        return out

    @staticmethod
    def kad_shard_plan(unit_tiles, shards: int) -> np.ndarray:
        """unit_tiles int64 [units] (each >= 1) -> int64 [shards + 1]: shard s = units [b[s], b[s + 1]) (host only)"""
        t = np.ascontiguousarray(unit_tiles, dtype=np.int64)
        bounds = np.empty(int(shards) + 1 if int(shards) >= 1 else 1, dtype=np.int64)
        _check(lib().fad_kad_shard_plan(t.ctypes.data, t.shape[0], int(shards), bounds.ctypes.data))
        return bounds

    # ------------------------------------------- precision, recall, density and coverage
    def knn_radii_sq(self, z: torch.Tensor, m: int, k: int) -> torch.Tensor:
        """z fp16 [m + n, d] (cuda, X rows first) -> fp32 [m + n] (cuda): the squared distance of each row of X to its
        k-th nearest other row of X, then the same for each row of Y within Y (fad_knn_radii_sq)."""
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        out = torch.empty(z.shape[0], dtype=torch.float32, device=z.device)
        _check(lib().fad_knn_radii_sq(self._h, z.data_ptr(), int(m), z.shape[0] - int(m), z.shape[1], int(k),
                                      out.data_ptr(), _stream()))
        return out

    def knn_radii_sq_sharded(self, z: torch.Tensor, m: int, k: int, local_shards: int = 0) -> torch.Tensor:
        """fad_knn_radii_sq_sharded: knn_radii_sq over shards (local_shards as for kad_sums_sharded)"""
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        out = torch.empty(z.shape[0], dtype=torch.float32, device=z.device)
        _check(lib().fad_knn_radii_sq_sharded(self._h, None, int(local_shards), z.data_ptr(), int(m), z.shape[0] - int(m),
                                              z.shape[1], int(k), out.data_ptr(), _stream()))
        return out

    def prdc_counts(self, z: torch.Tensor, m: int, radii_sq: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """z fp16 [m + n, d] (cuda, X rows first), radii_sq fp32 [m + n] (cuda) -> (inside int32 [n], flags uint8 [m])
        (cuda): the number of baseline balls that contain each y_j, and per x_i bit 0 = covered, bit 1 = recalled
        (fad_prdc_counts)."""
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        assert radii_sq.dtype == torch.float32 and radii_sq.is_cuda and radii_sq.is_contiguous()
        assert radii_sq.shape == (z.shape[0],)
        n = z.shape[0] - int(m)
        inside = torch.empty(max(n, 0), dtype=torch.int32, device=z.device)
        flags = torch.empty(max(int(m), 0), dtype=torch.uint8, device=z.device)
        _check(lib().fad_prdc_counts(self._h, z.data_ptr(), int(m), n, z.shape[1], radii_sq.data_ptr(),
                                     inside.data_ptr(), flags.data_ptr(), _stream()))
        return inside, flags

    def prdc_counts_sharded(self, z: torch.Tensor, m: int, radii_sq: torch.Tensor,
                            local_shards: int = 0) -> tuple[torch.Tensor, torch.Tensor]:
        """fad_prdc_counts_sharded: prdc_counts over shards (local_shards as for kad_sums_sharded)"""
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        assert radii_sq.dtype == torch.float32 and radii_sq.is_cuda and radii_sq.is_contiguous()
        assert radii_sq.shape == (z.shape[0],)
        n = z.shape[0] - int(m)
        inside = torch.empty(max(n, 0), dtype=torch.int32, device=z.device)
        flags = torch.empty(max(int(m), 0), dtype=torch.uint8, device=z.device)
        _check(lib().fad_prdc_counts_sharded(self._h, None, int(local_shards), z.data_ptr(), int(m), n, z.shape[1],
                                             radii_sq.data_ptr(), inside.data_ptr(), flags.data_ptr(), _stream()))
        return inside, flags

    # Per-song PRDC (include/fadtk_b200.h): z = [X; Y_1; ...] fp16 (cuda), offsets int64 [n_items + 1] (cuda, into the
    # rows after X)
    def knn_song_radii_sq(self, z: torch.Tensor, m: int, offsets: torch.Tensor, k: int) -> torch.Tensor:
        """-> fp32 [m + n_total] (cuda): r_i^2 within X, then s_j^2 of each row of Y within its own song
        (fad_knn_song_radii_sq)"""
        return self._song_radii(lib().fad_knn_song_radii_sq, (), z, m, offsets, k)

    def knn_song_radii_sq_sharded(self, z: torch.Tensor, m: int, offsets: torch.Tensor, k: int,
                                  local_shards: int = 0) -> torch.Tensor:
        """fad_knn_song_radii_sq_sharded: knn_song_radii_sq over shards (local_shards as for kad_sums_sharded)"""
        return self._song_radii(lib().fad_knn_song_radii_sq_sharded, (None, int(local_shards)), z, m, offsets, k)

    def _song_radii(self, fn, shard_args, z, m, offsets, k):
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous() and offsets.ndim == 1
        out = torch.empty(z.shape[0], dtype=torch.float32, device=z.device)
        _check(fn(self._h, *shard_args, z.data_ptr(), int(m), offsets.data_ptr(), offsets.shape[0] - 1, z.shape[1],
                  int(k), out.data_ptr(), _stream()))
        return out

    def prdc_song_counts(self, z: torch.Tensor, m: int, offsets: torch.Tensor,
                         radii_sq: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """radii_sq fp32 [m + n_total] (cuda) -> (inside int32 [n_total], song_counts int32 [n_items, 2]) (cuda): the
        baseline balls that contain each y_j, and per song the covered and recalled baseline rows
        (fad_prdc_song_counts)"""
        return self._song_counts(lib().fad_prdc_song_counts, (), z, m, offsets, radii_sq)

    def prdc_song_counts_sharded(self, z: torch.Tensor, m: int, offsets: torch.Tensor, radii_sq: torch.Tensor,
                                 local_shards: int = 0) -> tuple[torch.Tensor, torch.Tensor]:
        """fad_prdc_song_counts_sharded: prdc_song_counts over shards (local_shards as for kad_sums_sharded)"""
        return self._song_counts(lib().fad_prdc_song_counts_sharded, (None, int(local_shards)), z, m, offsets, radii_sq)

    def _song_counts(self, fn, shard_args, z, m, offsets, radii_sq):
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous() and offsets.ndim == 1
        assert radii_sq.dtype == torch.float32 and radii_sq.is_cuda and radii_sq.is_contiguous()
        assert radii_sq.shape == (z.shape[0],)
        n_items = offsets.shape[0] - 1
        inside = torch.empty(max(z.shape[0] - int(m), 0), dtype=torch.int32, device=z.device)
        counts = torch.empty((max(n_items, 0), 2), dtype=torch.int32, device=z.device)
        _check(fn(self._h, *shard_args, z.data_ptr(), int(m), offsets.data_ptr(), n_items, z.shape[1],
                  radii_sq.data_ptr(), inside.data_ptr(), counts.data_ptr(), _stream()))
        return inside, counts

    @staticmethod
    def prdc_song_spans(offsets, m: int) -> np.ndarray:
        """offsets int64 [n_items + 1] (host) -> int64 [spans, 4]: {first row, end row, first song, songs} of each span
        of the per-song counts pass against m baseline rows (fad_prdc_song_spans, host only)"""
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        n_items = max(off.shape[0] - 1, 0)
        spans = np.empty((max(n_items, 1), 4), dtype=np.int64)
        n = np.zeros(1, dtype=np.int64)
        _check(lib().fad_prdc_song_spans(off.ctypes.data, n_items, int(m), spans.ctypes.data, n.ctypes.data))
        return spans[:int(n[0])]

    # ------------------------------------------- per-sample realism and nearest baseline row
    def realism(self, z: torch.Tensor, m: int, k: int):
        """z fp16 [m + n, d] (cuda, X rows first) -> (kept_radii_sq fp32 [m], realism fp32 [n], nearest int32 [n],
        nearest_sq fp32 [n]) (cuda) and the threshold T (float): the pruned baseline radii, each eval row's realism
        score, and its nearest baseline row and squared distance (fad_realism)."""
        return self._realism(lib().fad_realism, (), z, m, k)

    def realism_sharded(self, z: torch.Tensor, m: int, k: int, local_shards: int = 0):
        """fad_realism_sharded: realism over shards (local_shards as for kad_sums_sharded)"""
        return self._realism(lib().fad_realism_sharded, (None, int(local_shards)), z, m, k)

    def _realism(self, fn, shard_args, z, m, k):
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        m, n = int(m), z.shape[0] - int(m)
        kept = torch.empty(max(m, 0), dtype=torch.float32, device=z.device)
        realism = torch.empty(max(n, 0), dtype=torch.float32, device=z.device)
        nearest = torch.empty(max(n, 0), dtype=torch.int32, device=z.device)
        nearest_sq = torch.empty(max(n, 0), dtype=torch.float32, device=z.device)
        t = C.c_double(0.0)
        _check(fn(self._h, *shard_args, z.data_ptr(), m, n, z.shape[1], int(k), kept.data_ptr(), realism.data_ptr(),
                  nearest.data_ptr(), nearest_sq.data_ptr(), C.addressof(t), _stream()))
        return kept, realism, nearest, nearest_sq, t.value

    # ------------------------------------------- k nearest distinct baseline groups
    def nearest(self, z: torch.Tensor, m: int, k: int, offsets: "torch.Tensor | None" = None):
        """z fp16 [m + n, d] (cuda, X rows first), offsets int64 [groups + 1] (cuda) or None (every baseline row its own
        group) -> (nearest int32 [n, k], nearest_sq fp32 [n, k]) (cuda): per eval row the k nearest distinct groups of
        X, each as the row and q of its nearest row, ascending; -1 / +inf past the last non-empty group (fad_nearest)."""
        return self._nearest(lib().fad_nearest, (), z, m, k, offsets)

    def nearest_sharded(self, z: torch.Tensor, m: int, k: int, offsets: "torch.Tensor | None" = None,
                        local_shards: int = 0):
        """fad_nearest_sharded: nearest over shards (local_shards as for kad_sums_sharded)"""
        return self._nearest(lib().fad_nearest_sharded, (None, int(local_shards)), z, m, k, offsets)

    def _nearest(self, fn, shard_args, z, m, k, offsets):
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        m, n = int(m), z.shape[0] - int(m)
        shape = (max(n, 0), max(int(k), 0))
        nearest = torch.empty(shape, dtype=torch.int32, device=z.device)
        nearest_sq = torch.empty(shape, dtype=torch.float32, device=z.device)
        if offsets is not None:
            assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous()
        off, groups = (None, 0) if offsets is None else (offsets.data_ptr(), offsets.numel() - 1)
        _check(fn(self._h, *shard_args, z.data_ptr(), m, n, z.shape[1], int(k), off, groups, nearest.data_ptr(),
                  nearest_sq.data_ptr(), _stream()))
        return nearest, nearest_sq

    # ------------------------------------------- permutation tests of KAD (DESIGN.md 5.16)
    # A pool of n rows, `a` of them labelled; labelling 0 marks rows 0 .. a - 1, labellings 1 .. B come from the seed
    # (include/fadtk_b200.h).  seed: an int in [0, 2**64).
    def perm_labels(self, n: int, a: int, labellings: int, seed: int) -> torch.Tensor:
        """-> int32 [B + 1, 4 ceil(n / 128)] (cuda; the uint32 words' bits): bit i & 31 of word i >> 5 of row b is row i's
        label in labelling b (fad_perm_labels)"""
        words = 4 * ((max(int(n), 0) + 127) // 128)
        out = torch.empty((max(int(labellings), 0) + 1, max(words, 4)), dtype=torch.int32, device=self.torch_device)
        _check(lib().fad_perm_labels(self._h, int(n), int(a), int(labellings), int(seed), out.data_ptr(), _stream()))
        return out

    def perm_dot(self, bits: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
        """bits as perm_labels gives them, v fp64 [n] (cuda) -> fp64 [B + 1] (cuda): per labelling the sum of v over the
        rows it marks, in a fixed order (fad_perm_dot)"""
        assert bits.dtype == torch.int32 and bits.is_cuda and bits.is_contiguous() and bits.ndim == 2
        assert v.dtype == torch.float64 and v.is_cuda and v.is_contiguous() and v.ndim == 1
        assert bits.shape[1] == 4 * ((v.shape[0] + 127) // 128)
        out = torch.empty(bits.shape[0], dtype=torch.float64, device=v.device)
        _check(lib().fad_perm_dot(self._h, bits.data_ptr(), v.shape[0], bits.shape[0] - 1, v.data_ptr(), out.data_ptr(),
                                  _stream()))
        return out

    def kad_perm_sums(self, z: torch.Tensor, a: int, sigma: torch.Tensor, labellings: int, seed: int) -> torch.Tensor:
        """z fp16 [n, d] (cuda, the pool), sigma fp64 scalar (cuda) -> fp64 [B + 1, 3] (cuda): (S_aa, S_bb, S_ab) of
        every labelling, each kernel value rounded to fp16 once (fad_kad_perm_sums)"""
        return self._perm_sums(lib().fad_kad_perm_sums, (), z, a, sigma, labellings, seed)

    def kad_perm_sums_sharded(self, z: torch.Tensor, a: int, sigma: torch.Tensor, labellings: int, seed: int,
                              local_shards: int = 0) -> torch.Tensor:
        """fad_kad_perm_sums_sharded: kad_perm_sums over shards (local_shards as for kad_sums_sharded)"""
        return self._perm_sums(lib().fad_kad_perm_sums_sharded, (None, int(local_shards)), z, a, sigma, labellings, seed)

    def _perm_sums(self, fn, shard_args, z, a, sigma, labellings, seed):
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        assert sigma.dtype == torch.float64 and sigma.is_cuda and sigma.numel() == 1
        out = torch.empty((max(int(labellings), 0) + 1, 3), dtype=torch.float64, device=z.device)
        _check(fn(self._h, *shard_args, z.data_ptr(), z.shape[0], int(a), z.shape[1], sigma.data_ptr(), int(labellings),
                  int(seed), out.data_ptr(), _stream()))
        return out

    # ------------------------------------- permutation test of the FAD difference (DESIGN.md 5.17)
    @staticmethod
    def record_len(d: int) -> int:
        """R(d) = 1 + d + d (d + 1) / 2: the fp64 values of one unit record (fad_record_len)"""
        return int(lib().fad_record_len(int(d)))

    def unit_records(self, emb: torch.Tensor, offsets: torch.Tensor, shift: torch.Tensor) -> torch.Tensor:
        """emb fp16 [N, d], offsets int64 [n_units + 1], shift fp16 [d] (all cuda) -> fp64 [n_units, R(d)] (cuda):
        per unit [n | sum y | upper triangle of sum y y^T], y = x - shift (fad_unit_records)"""
        assert emb.dtype == torch.float16 and emb.is_cuda and emb.is_contiguous() and emb.ndim == 2
        assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous() and offsets.ndim == 1
        assert shift.dtype == torch.float16 and shift.is_cuda and shift.is_contiguous()
        n_units, d = offsets.shape[0] - 1, emb.shape[1]
        out = torch.empty((max(n_units, 0), self.record_len(d)), dtype=torch.float64, device=emb.device)
        _check(lib().fad_unit_records(self._h, emb.data_ptr(), offsets.data_ptr(), n_units, d, shift.data_ptr(),
                                      out.data_ptr(), _stream()))
        return out

    def perm_record_sums(self, records: torch.Tensor, bits: torch.Tensor, d: int) -> torch.Tensor:
        """records fp64 [n_units, R(d)], bits as perm_labels(n_units, ...) gives them -> fp64 [B + 1, 2, R(d)] (cuda):
        per labelling the sums of the records of the units it marks and of the others (fad_perm_record_sums)"""
        assert records.dtype == torch.float64 and records.is_cuda and records.is_contiguous() and records.ndim == 2
        assert bits.dtype == torch.int32 and bits.is_cuda and bits.is_contiguous() and bits.ndim == 2
        out = torch.empty((bits.shape[0], 2, records.shape[1]), dtype=torch.float64, device=records.device)
        _check(lib().fad_perm_record_sums(self._h, records.data_ptr(), records.shape[0], int(d), bits.data_ptr(),
                                          bits.shape[0] - 1, out.data_ptr(), _stream()))
        return out

    # ------------------------------------------- bootstrap confidence intervals (DESIGN.md 5.18)
    # n_units units resampled B = resamples times; resample 0 is the observed set (include/fadtk_b200.h).
    def boot_counts(self, n_units: int, resamples: int, seed: int) -> torch.Tensor:
        """-> int32 [B + 1, n_units] (cuda; the uint32 multiplicities): how often resample b draws unit u
        (fad_boot_counts)"""
        out = torch.empty((max(int(resamples), 0) + 1, max(int(n_units), 1)), dtype=torch.int32, device=self.torch_device)
        _check(lib().fad_boot_counts(self._h, int(n_units), int(resamples), int(seed), out.data_ptr(), _stream()))
        return out

    def boot_record_sums(self, records: torch.Tensor, counts: torch.Tensor, d: int) -> torch.Tensor:
        """records fp64 [n_units, R(d)], counts as boot_counts(n_units, ...) gives them -> fp64 [B + 1, R(d)] (cuda): per
        resample the multiplicity-weighted sum of the records (fad_boot_record_sums)"""
        assert records.dtype == torch.float64 and records.is_cuda and records.is_contiguous() and records.ndim == 2
        assert counts.dtype == torch.int32 and counts.is_cuda and counts.is_contiguous() and counts.ndim == 2
        assert counts.shape[1] == records.shape[0]
        out = torch.empty((counts.shape[0], records.shape[1]), dtype=torch.float64, device=records.device)
        _check(lib().fad_boot_record_sums(self._h, records.data_ptr(), records.shape[0], int(d), counts.data_ptr(),
                                          counts.shape[0] - 1, out.data_ptr(), _stream()))
        return out

    def kad_boot_sums(self, y: torch.Tensor, offsets: torch.Tensor, sigma: torch.Tensor, g_units: torch.Tensor,
                      resamples: int, seed: int) -> torch.Tensor:
        """y fp16 [n, d] (cuda, the eval rows, d a multiple of 8), offsets int64 [n_units + 1], sigma fp64 scalar,
        g_units fp64 [n_units] (cuda) -> fp64 [B + 1, 3] (cuda): (n_b, S_yy(b), S_xy(b)) of every resample
        (fad_kad_boot_sums)"""
        assert y.dtype == torch.float16 and y.is_cuda and y.is_contiguous() and y.ndim == 2
        assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous() and offsets.ndim == 1
        assert sigma.dtype == torch.float64 and sigma.is_cuda and sigma.numel() == 1
        assert g_units.dtype == torch.float64 and g_units.is_cuda and g_units.is_contiguous()
        out = torch.empty((max(int(resamples), 0) + 1, 3), dtype=torch.float64, device=y.device)
        _check(lib().fad_kad_boot_sums(self._h, y.data_ptr(), offsets.data_ptr(), offsets.shape[0] - 1, y.shape[1],
                                       sigma.data_ptr(), g_units.data_ptr(), int(resamples), int(seed), out.data_ptr(),
                                       _stream()))
        return out

    # ------------------------------------------- a prepared baseline (DESIGN.md 5.15)
    # The _sharded forms take local_shards as kad_sums_sharded does; None runs the unsharded entry.
    def pair_digest(self, z: torch.Tensor) -> int:
        """z fp16 [rows, d] (cuda) -> the row digest the sharded entries compare (fad_pair_digest), as an int"""
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        out = torch.empty(1, dtype=torch.int64, device=z.device)
        _check(lib().fad_pair_digest(self._h, z.data_ptr(), z.shape[0], z.shape[1], out.data_ptr(), _stream()))
        return int(out.cpu().numpy().view(np.uint64)[0])

    def knn_lists_sq(self, x: torch.Tensor, k_max: int, local_shards: "int | None" = None) -> torch.Tensor:
        """x fp16 [m, d] (cuda) -> fp32 [m, k_max] (cuda): per row the k_max smallest q to the other rows, ascending
        (fad_knn_lists_sq, or fad_knn_lists_sq_sharded)"""
        assert x.dtype == torch.float16 and x.is_cuda and x.is_contiguous() and x.ndim == 2
        out = torch.empty((x.shape[0], max(int(k_max), 0)), dtype=torch.float32, device=x.device)
        fn, sa = _prepared_fn("fad_knn_lists_sq", local_shards)
        _check(fn(self._h, *sa, x.data_ptr(), x.shape[0], x.shape[1], int(k_max), out.data_ptr(), _stream()))
        return out

    def kad_eval_sums(self, z: torch.Tensor, m: int, offsets: torch.Tensor, sigma: torch.Tensor,
                      local_shards: "int | None" = None) -> torch.Tensor:
        """kad_song_sums without S_xx -> fp64 [n_items, 2] (cuda): S_yy,k, S_xy,k per item (fad_kad_eval_sums)"""
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous() and offsets.ndim == 1
        assert sigma.dtype == torch.float64 and sigma.is_cuda and sigma.numel() == 1
        n_items = offsets.shape[0] - 1
        out = torch.empty((max(n_items, 0), 2), dtype=torch.float64, device=z.device)
        fn, sa = _prepared_fn("fad_kad_eval_sums", local_shards)
        _check(fn(self._h, *sa, z.data_ptr(), int(m), offsets.data_ptr(), n_items, z.shape[1], sigma.data_ptr(),
                  out.data_ptr(), _stream()))
        return out

    def knn_eval_radii_sq(self, z: torch.Tensor, m: int, k: int, offsets: "torch.Tensor | None" = None,
                          local_shards: "int | None" = None) -> torch.Tensor:
        """z fp16 [m + n, d] (cuda, X rows first) -> fp32 [n] (cuda): s_j^2 of each eval row within the eval set, or
        within its own song when offsets (int64 [n_items + 1], cuda) are given (fad_knn_eval_radii_sq)"""
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        n = z.shape[0] - int(m)
        if offsets is None:
            off, n_items = None, n
        else:
            assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous() and offsets.ndim == 1
            off, n_items = offsets.data_ptr(), offsets.shape[0] - 1
        out = torch.empty(max(n, 0), dtype=torch.float32, device=z.device)
        fn, sa = _prepared_fn("fad_knn_eval_radii_sq", local_shards)
        _check(fn(self._h, *sa, z.data_ptr(), int(m), off, n_items, z.shape[1], int(k), out.data_ptr(), _stream()))
        return out

    def realism_prepared(self, z: torch.Tensor, m: int, kept_radii_sq: torch.Tensor,
                         local_shards: "int | None" = None):
        """z fp16 [m + n, d] (cuda, X rows first), kept_radii_sq fp32 [m] (cuda) -> (realism fp32 [n], nearest int32
        [n], nearest_sq fp32 [n]) (cuda): fad_realism's tile pass alone (fad_realism_prepared)"""
        assert z.dtype == torch.float16 and z.is_cuda and z.is_contiguous() and z.ndim == 2
        assert kept_radii_sq.dtype == torch.float32 and kept_radii_sq.is_cuda and kept_radii_sq.is_contiguous()
        m, n = int(m), z.shape[0] - int(m)
        realism = torch.empty(max(n, 0), dtype=torch.float32, device=z.device)
        nearest = torch.empty(max(n, 0), dtype=torch.int32, device=z.device)
        nearest_sq = torch.empty(max(n, 0), dtype=torch.float32, device=z.device)
        fn, sa = _prepared_fn("fad_realism_prepared", local_shards)
        _check(fn(self._h, *sa, z.data_ptr(), m, n, z.shape[1], kept_radii_sq.data_ptr(), realism.data_ptr(),
                  nearest.data_ptr(), nearest_sq.data_ptr(), _stream()))
        return realism, nearest, nearest_sq


_build_id = None


def build_id() -> str:
    """sha1 of the loaded library file: a saved preparation is trusted only by the build that wrote it"""
    global _build_id
    if _build_id is None:
        import hashlib
        _build_id = hashlib.sha1(_LIB_PATH.read_bytes()).hexdigest()
    return _build_id


def _prepared_fn(name: str, local_shards):
    """the entry `name` and its extra arguments: unsharded (local_shards None), else its _sharded form"""
    if local_shards is None:
        return getattr(lib(), name), ()
    return getattr(lib(), name + "_sharded"), (None, int(local_shards))


class Baseline:
    """Device-resident baseline statistics with the matrix square root precomputed."""

    def __init__(self, eng: "Engine", mu, cov):
        dev = eng.torch_device
        self.eng = eng
        def to_dev(a):
            if isinstance(a, torch.Tensor):
                return a.to(dev, torch.float64).contiguous()
            return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64)).to(dev)
        self.mu = to_dev(mu)
        cov = to_dev(cov)
        self.d = self.mu.shape[0]
        self.sqrt = torch.empty((self.d, self.d), dtype=torch.float64, device=dev)
        self.scal = torch.empty(2, dtype=torch.float64, device=dev)
        _check(lib().fad_sqrt_psd(eng._h, cov.data_ptr(), self.d, 0, self.sqrt.data_ptr(), self.scal.data_ptr(), _stream()))

    def frechet(self, mu2: torch.Tensor, cov2: torch.Tensor) -> torch.Tensor:
        """fp64 device tensors -> fp64 [8] device (same layout as Engine.frechet)."""
        out = torch.zeros(8, dtype=torch.float64, device=self.mu.device)
        _check(lib().fad_frechet_presqrt(self.eng._h, self.mu.data_ptr(), self.sqrt.data_ptr(), self.scal.data_ptr(),
                                         mu2.data_ptr(), cov2.data_ptr(), self.d, 0, out.data_ptr(), _stream()))
        return out

    def frechet_batched(self, emb: torch.Tensor, offsets: torch.Tensor) -> torch.Tensor:
        """emb fp16 [N, d], offsets int64 [n_items + 1] (both cuda) -> fp64 [n_items, 8]: every item's
        FAD against this baseline in one lock-step launch sequence (fad_frechet_batched)."""
        assert emb.dtype == torch.float16 and emb.is_cuda and emb.is_contiguous() and emb.shape[1] == self.d
        assert offsets.dtype == torch.int64 and offsets.is_cuda
        n_items = offsets.shape[0] - 1
        out = torch.zeros((n_items, 8), dtype=torch.float64, device=emb.device)
        _check(lib().fad_frechet_batched(self.eng._h, self.mu.data_ptr(), self.sqrt.data_ptr(), self.scal.data_ptr(),
                                         emb.data_ptr(), offsets.data_ptr(), n_items, self.d, 0, out.data_ptr(), _stream()))
        return out


    def frechet_records(self, sums: torch.Tensor, shift: torch.Tensor) -> torch.Tensor:
        """sums fp64 [..., R(d)] (cuda, e.g. perm_record_sums' output), shift fp16 [d] -> fp64 [..., 8]: the FAD of
        each sum's mean and covariance against this baseline, [7] = its row count (fad_frechet_records)"""
        assert sums.dtype == torch.float64 and sums.is_cuda and sums.is_contiguous()
        assert shift.dtype == torch.float16 and shift.is_cuda and shift.is_contiguous()
        items = sums.numel() // sums.shape[-1]
        out = torch.empty((*sums.shape[:-1], 8), dtype=torch.float64, device=sums.device)
        _check(lib().fad_frechet_records(self.eng._h, self.mu.data_ptr(), self.sqrt.data_ptr(), self.scal.data_ptr(),
                                         sums.data_ptr(), items, self.d, shift.data_ptr(), 0, out.data_ptr(), _stream()))
        return out

    def frechet_perm(self, emb: torch.Tensor, offsets: torch.Tensor, a: int, labellings: int, seed: int):
        """emb fp16 [N, d], offsets int64 [n_units + 1] (cuda; units 0 .. a - 1 are system A's) -> (fp64
        [B + 1, 2, 8], the fp16 shift [d] used) (cuda): the FAD of both sides of every labelling (fad_frechet_perm)"""
        assert emb.dtype == torch.float16 and emb.is_cuda and emb.is_contiguous() and emb.shape[1] == self.d
        assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous() and offsets.ndim == 1
        out = torch.empty((max(int(labellings), 0) + 1, 2, 8), dtype=torch.float64, device=emb.device)
        shift = torch.empty(self.d, dtype=torch.float16, device=emb.device)
        _check(lib().fad_frechet_perm(self.eng._h, self.mu.data_ptr(), self.sqrt.data_ptr(), self.scal.data_ptr(),
                                      emb.data_ptr(), offsets.data_ptr(), offsets.shape[0] - 1, int(a), self.d,
                                      int(labellings), int(seed), 0, shift.data_ptr(), out.data_ptr(), _stream()))
        return out, shift

    def frechet_boot(self, emb: torch.Tensor, offsets: torch.Tensor, resamples: int, seed: int):
        """emb fp16 [N, d], offsets int64 [n_units + 1] (cuda) -> (fp64 [B + 1, 8], the fp16 shift [d] used) (cuda): the
        FAD of every bootstrap resample of the units, resample 0 the observed set (fad_frechet_boot)"""
        assert emb.dtype == torch.float16 and emb.is_cuda and emb.is_contiguous() and emb.shape[1] == self.d
        assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous() and offsets.ndim == 1
        out = torch.empty((max(int(resamples), 0) + 1, 8), dtype=torch.float64, device=emb.device)
        shift = torch.empty(self.d, dtype=torch.float16, device=emb.device)
        _check(lib().fad_frechet_boot(self.eng._h, self.mu.data_ptr(), self.sqrt.data_ptr(), self.scal.data_ptr(),
                                      emb.data_ptr(), offsets.data_ptr(), offsets.shape[0] - 1, self.d, int(resamples),
                                      int(seed), 0, shift.data_ptr(), out.data_ptr(), _stream()))
        return out, shift


class PairwiseBaseline:
    """A prepared baseline for the pairwise metrics (DESIGN.md 5.15): the baseline rows X on the device and what depends
    on them alone, computed once - the row digest (fad_pair_digest), the KAD bandwidth (the two middle q of the xx pairs
    and sigma), S_xx (fad_kad_song_sums with no songs), and per row the k_max smallest q to the other rows
    (fad_knn_lists_sq).  KAD, PRDC (k <= k_max), realism (k <= k_max) and nearest then pay for the eval rows only.
    x: fp16 [m, d] (cuda, d a multiple of 8); d_orig: the width before zero-padding; offsets: int64 [files + 1] of the
    baseline's files, or None; local_shards as for Engine.knn_lists_sq.  sigma is 0 and s_xx NaN when more than half of
    the baseline pairs are identical rows (KAD refuses such a baseline, PRDC does not need them)."""
    VERSION = 1

    def __init__(self, eng: "Engine", x: torch.Tensor, k_max: int, d_orig: int, offsets=None,
                 local_shards: "int | None" = None, _state: "dict | None" = None):
        assert x.dtype == torch.float16 and x.is_contiguous() and x.ndim == 2
        self.eng, self.x, self.k_max, self.d = eng, x, int(k_max), int(d_orig)
        self.m = int(x.shape[0])
        self.offsets = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.int64)
        self._kept: dict = {}
        self.digest = eng.pair_digest(x)
        if _state is not None:
            self.median_sq = np.asarray(_state["median_sq"], dtype=np.float64)
            self.sigma, self.s_xx = float(_state["sigma"]), float(_state["s_xx"])
            self.lists = torch.from_numpy(np.ascontiguousarray(_state["lists"], dtype=np.float32)).to(x.device)
            return
        sh = () if local_shards is None else (int(local_shards),)
        self.median_sq = (eng.kad_median_sq_sharded(x, *sh) if sh else eng.kad_median_sq(x)).cpu().numpy()
        self.sigma = 0.5 * (float(np.sqrt(self.median_sq[0])) + float(np.sqrt(self.median_sq[1])))
        self.s_xx = float("nan")
        if self.sigma > 0.0:
            none = torch.zeros(1, dtype=torch.int64, device=x.device)
            sig = torch.tensor([self.sigma], dtype=torch.float64, device=x.device)
            sums = eng.kad_song_sums_sharded(x, self.m, none, sig, *sh) if sh else eng.kad_song_sums(x, self.m, none, sig)
            self.s_xx = float(sums.cpu().numpy()[0])
        self.lists = eng.knn_lists_sq(x, self.k_max, local_shards)

    def kept_radii(self, k: int):
        """-> (kept radii fp32 [m] (cuda), T) of realism at k <= k_max, by fad_realism's rule: r_i^2 = list column
        k - 1, T = their numpy.median in fp64, r~_i^2 = r_i^2 where r_i^2 <= T, else 0"""
        if k not in self._kept:
            r = self.lists[:, k - 1].contiguous()
            h = np.sort(r.cpu().numpy().astype(np.float64))
            mid = self.m // 2
            t = float(h[mid]) if self.m % 2 else float((h[mid - 1] + h[mid]) / 2.0)
            self._kept[k] = (torch.where(r.double() <= t, r, torch.zeros_like(r)), t)
        return self._kept[k]

    def save(self, path, fingerprint: dict) -> None:
        """Write the preparation to path (.npz) atomically: a temporary file in the same directory, then os.replace."""
        path = Path(path)
        path.parent.mkdir(parents=True, exist_ok=True)
        tmp = path.with_name(path.name + f".tmp{os.getpid()}")
        with open(tmp, "wb") as fh:
            np.savez(fh, version=np.int64(self.VERSION), build=np.array(build_id()), m=np.int64(self.m),
                     d=np.int64(self.d), k_max=np.int64(self.k_max), digest=np.uint64(self.digest),
                     median_sq=self.median_sq, sigma=np.float64(self.sigma), s_xx=np.float64(self.s_xx),
                     lists=self.lists.cpu().numpy(),
                     offsets=self.offsets if self.offsets is not None else np.zeros(0, dtype=np.int64),
                     fingerprint=np.array(json.dumps(fingerprint, sort_keys=True)))
        os.replace(tmp, path)

    @classmethod
    def load(cls, path, eng: "Engine", x: torch.Tensor, k_max: int, d_orig: int, fingerprint: dict, offsets=None):
        """-> (PairwiseBaseline, "") when the file at path was written for these rows by this build: the same format
        version and library (build_id), m, d, k_max >= the one asked for, the fingerprint of the embedding files and the digest of x;
        else (None, why it is not used).  x, d_orig, offsets as for the constructor."""
        path = Path(path)
        if not path.exists():
            return None, "no saved preparation"
        try:
            with np.load(path, allow_pickle=False) as f:
                st = {k: f[k] for k in f.files}
            if int(st["version"]) != cls.VERSION:
                return None, f"its format version is {int(st['version'])}, not {cls.VERSION}"
            if str(st["build"]) != build_id():
                return None, "another build of the library wrote it"
            if json.loads(str(st["fingerprint"])) != fingerprint:
                return None, "the embedding files changed"
            for key, v in (("m", int(x.shape[0])), ("d", int(d_orig))):
                if int(st[key]) != v:
                    return None, f"its {key} is {int(st[key])}, not {v}"
            if int(st["k_max"]) < int(k_max):
                return None, f"its k_max is {int(st['k_max'])}, below {int(k_max)}"
            if st["lists"].shape != (int(x.shape[0]), int(st["k_max"])) or st["lists"].dtype != np.float32:
                return None, "its radius lists have the wrong shape"
            off = None if offsets is None else np.asarray(offsets, dtype=np.int64)
            if (off is None and st["offsets"].size) or (off is not None and not np.array_equal(off, st["offsets"])):
                return None, "the file offsets differ"
        except (OSError, ValueError, KeyError) as e:
            return None, f"it cannot be read ({e})"
        pb = cls(eng, x, int(st["k_max"]), d_orig, offsets, _state=st)
        if pb.digest != int(st["digest"]):
            return None, "the rows on the device differ from the ones it was computed from"
        return pb, ""


_engines: dict = {}


def engine(device: int | None = None, max_examples: int | None = None) -> Engine:
    """Process-wide engine per device (created lazily)."""
    dev = torch.cuda.current_device() if device is None else int(device)
    if dev not in _engines:
        me = max_examples or int(os.environ.get("FADTK_MAX_EXAMPLES", "2048"))
        _engines[dev] = Engine(dev, me)
    return _engines[dev]
