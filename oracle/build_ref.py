#!/usr/bin/env python3
"""Recipe for oracle/_ref: the UNMODIFIED reference encoder modules, copied from where they lie under
/root/reference into the git-ignored directory oracle/_ref/ so that they travel to the GPU box with the snapshot.

TEST / MEASUREMENT INFRASTRUCTURE ONLY (never imported by auto_avsr_b200).  The reference is pure Python, so "building"
it is a file copy; nothing is edited and nothing under oracle/_ref is committed (.gitignore).  Users:
  * bench.py --impl reference and bench.py's cpu_baseline leg time THIS code (kind "reference") on the host cores;
  * tests/test_oracle_golden.py::test_ref_copy_reproduces_golden checks the copy against the committed fixtures;
  * tests/test_boundary_cpu.py and tests/test_decoder_dropin_cpu.py drive the drop-ins from the reference's own modules.
Run:  python oracle/build_ref.py [/root/reference]
"""
import filecmp
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, "_ref")
#: the files SURVEY.md section 8a cites (+ nets_utils for rename_state_dict / make_non_pad_mask, + the CTC head of 8f #1)
FILES = [
    "espnet/nets/pytorch_backend/encoder/conformer_encoder.py",
    "espnet/nets/pytorch_backend/transformer/__init__.py",
    "espnet/nets/pytorch_backend/transformer/attention.py",
    "espnet/nets/pytorch_backend/transformer/embedding.py",
    "espnet/nets/pytorch_backend/transformer/layer_norm.py",
    "espnet/nets/pytorch_backend/transformer/positionwise_feed_forward.py",
    "espnet/nets/pytorch_backend/transformer/repeat.py",
    "espnet/nets/pytorch_backend/nets_utils.py",
    "espnet/nets/pytorch_backend/ctc.py",
    # SURVEY.md 8f #3: the attention decoder, the CTC prefix scorer and the beam search that drives them
    "espnet/nets/pytorch_backend/decoder/transformer_decoder.py",
    "espnet/nets/pytorch_backend/transformer/mask.py",
    "espnet/nets/scorer_interface.py",
    "espnet/nets/scorers/__init__.py",
    "espnet/nets/scorers/ctc.py",
    "espnet/nets/scorers/length_bonus.py",
    "espnet/nets/ctc_prefix_score.py",
    "espnet/nets/e2e_asr_common.py",
    "espnet/nets/beam_search.py",
    "espnet/nets/batch_beam_search.py",
    # the E2E model that builds the encoder / CTC head (tests/test_boundary_cpu.py: install() / install_head())
    "espnet/nets/pytorch_backend/e2e_asr_conformer.py",
    "espnet/nets/pytorch_backend/frontend/resnet.py",
    "espnet/nets/pytorch_backend/frontend/resnet1d.py",
    "espnet/nets/pytorch_backend/transformer/add_sos_eos.py",
    "espnet/nets/pytorch_backend/transformer/label_smoothing_loss.py",
]


def build(src_root: str = "/root/reference") -> bool:
    """Copy the files; returns False (and leaves any existing copy alone) when the reference tree is absent."""
    if not os.path.isdir(os.path.join(src_root, "espnet")):
        return os.path.isdir(os.path.join(DST, "espnet"))
    for rel in FILES:
        src, dst = os.path.join(src_root, rel), os.path.join(DST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if not (os.path.exists(dst) and filecmp.cmp(src, dst, shallow=False)):
            shutil.copyfile(src, dst)
    with open(os.path.join(DST, "SOURCE.txt"), "w") as f:
        f.write(f"verbatim copies from {src_root} (mpc001/auto_avsr @ 182b628) made by oracle/build_ref.py:\n")
        f.writelines(rel + "\n" for rel in FILES)
    return True


def available() -> bool:
    return os.path.exists(os.path.join(DST, FILES[0]))


def import_reference_encoder():
    """-> (ConformerEncoder class, make_non_pad_mask) of the reference copy; raises ImportError if it was not built."""
    if not available():
        raise ImportError("oracle/_ref is not built (python oracle/build_ref.py in the build container)")
    if DST not in sys.path:
        sys.path.insert(0, DST)
    from espnet.nets.pytorch_backend.encoder import conformer_encoder as ce
    from espnet.nets.pytorch_backend.nets_utils import make_non_pad_mask
    if not os.path.abspath(ce.__file__).startswith(DST):
        raise ImportError(f"another espnet is already imported ({ce.__file__}); import the reference copy first")
    ConformerEncoder = ce.ConformerEncoder
    return ConformerEncoder, make_non_pad_mask


def import_reference_search():
    """-> dict of the reference copy's decoding classes (TransformerDecoder, CTC, CTCPrefixScorer, LengthBonus,
    BatchBeamSearch); raises ImportError if oracle/_ref was not built."""
    import_reference_encoder()
    from espnet.nets.batch_beam_search import BatchBeamSearch
    from espnet.nets.pytorch_backend.ctc import CTC
    from espnet.nets.pytorch_backend.decoder.transformer_decoder import TransformerDecoder
    from espnet.nets.scorers.ctc import CTCPrefixScorer
    from espnet.nets.scorers.length_bonus import LengthBonus
    return dict(TransformerDecoder=TransformerDecoder, CTC=CTC, CTCPrefixScorer=CTCPrefixScorer, LengthBonus=LengthBonus,
                BatchBeamSearch=BatchBeamSearch)


if __name__ == "__main__":
    ok = build(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
    print("oracle/_ref:", "ready" if ok else "reference tree not found, nothing copied")
