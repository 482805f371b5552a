"""Which GEMM callers may load their weight before the PDL dependency wait (EpiParams::b_static, gemm_tc.cu).

A GEMM with the flag reads its weight before griddepcontrol.wait, which is only safe when no kernel of the PDL chain
it runs in writes that weight.  The encoder forward (forward_body, compute_pos) and its head (proj_encoder, ctc_lo)
read prepared weights that avsr_prepare_weights wrote before the chain started; every other caller (the per-op
entries, the decoder, training, the front-ends) must leave the flag off.  The v^T GEMM has the weight in A and is
never flagged."""
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "auto_avsr_b200", "csrc")


def read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def function_body(src, name):
    """the text of `static int name(...) { ... }` (brace matched)"""
    m = re.search(r"static int " + name + r"\(", src)
    assert m, name
    i = src.index("{", m.end())
    depth = 0
    for j in range(i, len(src)):
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        if depth == 0:
            return src[i:j + 1]
    raise AssertionError(name)


def test_only_the_encoder_forward_sets_the_flag():
    for name in os.listdir(CSRC):
        if name.endswith(".cu") and name not in ("encoder.cu", "gemm_tc.cu"):
            src = read(name)
            assert "b_static" not in src and "static_b(" not in src, name
    enc = read("encoder.cu")
    flagged = {fn for fn in ("forward_body", "compute_pos", "head_forward_body", "ctc_logprobs")
               if "static_b(" in function_body(enc, fn) or "b_static" in function_body(enc, fn)}
    assert flagged == {"forward_body", "compute_pos", "head_forward_body", "ctc_logprobs"}
    # every gemm call of the encoder forward is flagged except v^T (weight in A)
    body = function_body(enc, "forward_body")
    calls = re.findall(r"run_gemm\(prec, (EPI_\w+), [^;]*;", body)
    assert len(calls) == 10, calls
    for call in re.finditer(r"run_gemm\(prec, (EPI_\w+), [^;]*;", body):
        assert ("static_b(" in call.group(0)) == (call.group(1) != "EPI_VT"), call.group(0)
    # ctc_lo is flagged only from the head forward, not from the per-op avsr_ctc_logprobs entry
    assert re.search(r"ctc_logprobs\([^;]*, true\);", function_body(enc, "head_forward_body"))
    assert "bool b_static = false" in enc
    # the per-op entries and the rest of the file do not set it
    outside = enc
    for fn in ("forward_body", "compute_pos", "head_forward_body", "ctc_logprobs"):
        outside = outside.replace(function_body(enc, fn), "")
    assert outside.count("static_b(") == 1        # the helper's own definition


def test_kernel_gates_the_prologue():
    src = read("gemm_tc.cu")
    # cluster launches and the v^T mode never take it; the kill switch clears the flag before dispatch
    assert "const bool pre = CS == 1 && MODE != EPI_VT && ep.b_static != 0;" in src
    assert 'getenv("AVSR_B200_PROLOGUE")' in src
    # the producer's barrier protocol is unchanged: a prologue stage is armed with the whole stage's bytes
    assert "mbar_expect_tx(full_bar(pre_its), Cfg::kStageBytes);" in src
