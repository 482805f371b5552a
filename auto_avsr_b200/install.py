"""Make the reference pick up the CUDA encoder without touching its sources.

``auto_avsr_b200.install()`` registers this package's modules under the reference's import paths, so
``from espnet.nets.pytorch_backend.encoder.conformer_encoder import ConformerEncoder``
(e2e_asr_conformer.py:12) resolves to the CUDA implementation and train.py / eval.py / lightning.py keep
driving it unchanged.  Call it before importing ``espnet.nets.pytorch_backend.e2e_asr_conformer`` (or after:
already-imported E2E modules get their ``ConformerEncoder`` symbol re-pointed).
"""
import sys
import types

REF_ENCODER_MODULE = "espnet.nets.pytorch_backend.encoder.conformer_encoder"
ALIAS_PACKAGE = "espnet.nets.pytorch_backend.conformer"          # north_star spelling (SURVEY.md D1)
E2E_MODULE = "espnet.nets.pytorch_backend.e2e_asr_conformer"


def install() -> None:
    from .espnet_dropin import conformer_encoder as ce
    from . import espnet_dropin as pkg

    sys.modules[REF_ENCODER_MODULE] = ce
    parent = sys.modules.get(REF_ENCODER_MODULE.rsplit(".", 1)[0])
    if parent is not None:
        setattr(parent, "conformer_encoder", ce)

    alias_pkg = types.ModuleType(ALIAS_PACKAGE)
    alias_pkg.__path__ = []                                    # mark as package
    alias_enc = types.ModuleType(ALIAS_PACKAGE + ".encoder")
    for name in ("Encoder", "ConformerEncoder", "EncoderLayer", "ConvolutionModule",
                 "RelPositionMultiHeadedAttention", "PositionwiseFeedForward", "LayerNorm"):
        setattr(alias_enc, name, getattr(pkg, name))
    alias_pkg.encoder = alias_enc
    sys.modules[ALIAS_PACKAGE] = alias_pkg
    sys.modules[ALIAS_PACKAGE + ".encoder"] = alias_enc

    e2e = sys.modules.get(E2E_MODULE)
    if e2e is not None:
        e2e.ConformerEncoder = ce.ConformerEncoder


def install_head(model):
    """The steps either side of the encoder (SURVEY.md 8f #1).  The reference builds ``proj_encoder`` as a bare
    ``torch.nn.Linear`` and ``ctc`` from a module it imports by name (e2e_asr_conformer.py:11, :31, :56), so instead of
    shadowing an import this re-homes the two sub-modules of an existing ``E2E`` instance: the drop-ins take over the
    very same ``Parameter`` objects (state dict, optimizer and checkpoint loading are unaffected)."""
    from .espnet_dropin.ctc import CTC, ProjEncoder

    old = model.proj_encoder
    new = ProjEncoder(old.in_features, old.out_features, bias=old.bias is not None)
    new.weight, new.bias = old.weight, old.bias
    new.train(old.training)
    model.proj_encoder = new

    oc = model.ctc
    nc = CTC(oc.ctc_lo.out_features, oc.ctc_lo.in_features, oc.dropout_rate, reduce=oc.reduce)
    nc.ctc_lo.weight, nc.ctc_lo.bias = oc.ctc_lo.weight, oc.ctc_lo.bias
    nc.train(oc.training)
    model.ctc = nc
    return model


def install_decoder(model):
    """The attention decoder's scoring path and the CTC prefix scorer (SURVEY.md 8f #3).  ``E2E`` builds its decoder from
    a class it imports by name and ``E2E.scorers()`` builds the CTC scorer likewise (e2e_asr_conformer.py:13,17,41-47,58-59):
    this re-homes the decoder of an existing ``E2E`` instance onto the drop-in (the very same ``Parameter`` objects) and
    re-points the two names in the already-imported E2E module, so ``model.scorers()`` -- what
    ``get_beam_search_decoder`` feeds to ``BatchBeamSearch`` (lightning.py:126-157) -- returns the CUDA scorers.
    Inference only: the teacher-forced ``decoder.forward`` of the training loss stays with the reference module, so call
    this on a model that is used for decoding."""
    from .espnet_dropin import scorer_interface, scorers_ctc
    from .espnet_dropin import transformer_decoder as td

    scorer_interface.rebind()
    old = model.decoder
    emb, first = old.embed[0], old.decoders[0]
    new = td.TransformerDecoder(odim=emb.num_embeddings, attention_dim=emb.embedding_dim, attention_heads=first.self_attn.h,
                                linear_units=first.feed_forward.w_1.out_features, num_blocks=len(old.decoders))
    for name, p in old.named_parameters():
        mod = new
        *path, leaf = name.split(".")
        for part in path:
            mod = getattr(mod, part) if not part.isdigit() else mod[int(part)]
        setattr(mod, leaf, p)
    new.train(old.training)
    model.decoder = new
    e2e = sys.modules.get(E2E_MODULE)
    if e2e is not None:
        e2e.TransformerDecoder = td.TransformerDecoder
        e2e.CTCPrefixScorer = scorers_ctc.CTCPrefixScorer
    return model


def is_installed() -> bool:
    mod = sys.modules.get(REF_ENCODER_MODULE)
    return mod is not None and mod.__name__.startswith("auto_avsr_b200")
