"""Every kernel-level entry point (extern "C" vqa_op_* in csrc/vqa_b200.cu) launches through glue_launch, that is through the Forward and
the stage functions the model forwards call, and never restates a launch itself. The kernel-level GPU suites are parity evidence for the
forwards only while both launch a kernel the same way. No GPU needed: this reads the source."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "t2v_metrics_b200", "csrc", "vqa_b200.cu")

# a raw launch, the GEMM / attention / norm dispatchers the Forward wraps (launch_attn_tc is the head-dim-64 launcher; the head-dim-128
# entries run launch_attn_tc128 inside f.attention)
DIRECT = [r"<<<", r"\brun_gemm\(", r"\blaunch_attn_tc\b", r"\blaunch_decode_attn\b", r"\brun_rmsnorm\b", r"\brun_layernorm"]


def op_bodies(text):
    """{name: body} of every extern "C" vqa_op_* definition, comments and string literals blanked."""
    text = re.sub(r"//[^\n]*|/\*.*?\*/", "", text, flags=re.S).replace('extern "C"', "EXTERN_C")
    text = re.sub(r'"(?:\\.|[^"\\])*"', '""', text)
    bodies = {}
    for m in re.finditer(r"EXTERN_C[^;{]*?\b(vqa_op_\w+)\s*\(", text):
        i = text.index("{", m.end())
        depth, j = 0, i
        while True:
            depth += {"{": 1, "}": -1}.get(text[j], 0)
            j += 1
            if depth == 0:
                break
        bodies[m.group(1)] = text[i:j]
    return bodies


def offenders(text):
    bad = {}
    for name, body in op_bodies(text).items():
        why = [p for p in DIRECT if re.search(p, body)]
        if "glue_launch(" not in body:
            why.append("no glue_launch")
        if why:
            bad[name] = why
    return bad


def test_every_kernel_entry_point_launches_through_the_forward_stages():
    text = open(SRC).read()
    assert len(op_bodies(text)) >= 31
    assert offenders(text) == {}

