"""H100-native (sm_90a) Conformer-encoder forward path for mpc001/auto_avsr (hot path only).

    import auto_avsr_b200; auto_avsr_b200.install()      # before importing the reference's E2E
    from auto_avsr_b200 import ConformerEncoder           # or use the class directly

Importing the compute modules requires the built CUDA library (``__graft_entry__.build()``); there is no
CPU or PyTorch fallback.  ``auto_avsr_b200.synthetic`` (weights / inputs generators) imports without it.
"""
__version__ = "0.1.0"

_LAZY = {"ConformerEncoder", "Encoder", "EncoderLayer", "ConvolutionModule", "RelPositionMultiHeadedAttention",
         "PositionwiseFeedForward", "LayerNorm", "RelPositionalEncoding", "CTC", "ProjEncoder", "TransformerDecoder",
         "CTCPrefixScorer", "LabelSmoothingLoss", "Conv3dResNet", "Conv1dResNet"}


def install():
    from .install import install as _install
    _install()


def install_head(model):
    """Swap an already-built reference ``E2E``'s ``proj_encoder`` and ``ctc`` for the CUDA drop-ins (same parameters)."""
    from .install import install_head as _install_head
    return _install_head(model)


def install_decoder(model):
    """Swap an already-built reference ``E2E``'s attention decoder (and ``criterion``) for the CUDA drop-ins and make
    ``model.scorers()`` return the CUDA CTC prefix scorer: the decoder then trains (teacher-forced forward + backward,
    LabelSmoothingLoss), validates and decodes in libavsr_b200."""
    from .install import install_decoder as _install_decoder
    return _install_decoder(model)


def install_frontend(model, library_train: bool = False):
    """Swap an already-built reference ``E2E``'s ResNet front-end for the CUDA drop-in (same parameters and buffers):
    in eval the front-end then runs in libavsr_b200 from the raw clip or waveform; with ``library_train`` its training
    forward and backward do too."""
    from .install import install_frontend as _install_frontend
    return _install_frontend(model, library_train=library_train)


def __getattr__(name):
    if name in _LAZY:
        from . import espnet_dropin
        return getattr(espnet_dropin, name)
    raise AttributeError(name)
