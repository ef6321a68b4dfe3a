#!/usr/bin/env python
"""Golden data of the robustness evaluation, produced by EXECUTING the reference's own code
(mce/eval_robustness.py, by its AST) from a checkout of the original project:

    python tests/golden/make_robustness_golden.py REFERENCE_DIR   # rewrites robustness_golden.json

It records
  * ALEXNET_CE, in the table's order (the module-level assignment, executed);
  * for 1..8 GPUs, the distortions each GPU's thread evaluates: process() is run for every thread index
    with FLAGS.gpu_index listing that many GPUs and show_corruption_error_by_distortion replaced by a
    recorder;
  * get_synsets2idx on a synthetic label file with spaces, capitals and surrounding blanks
    (tf.gfile.GFile stubbed with open).
tests/test_robustness_cpu.py checks the product against this file; it does not need the original project.
"""
import ast
import json
import os
import sys
import tempfile
import types

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "robustness_golden.json")
REL = os.path.join("mce", "eval_robustness.py")

LABEL_LINES = ["tench, Tinca tinca\n", "Goldfish\n", "  great white shark \n", "n01491361\n",
               "Tiger Shark, Galeocerdo Cuvieri\n", "HAMMERHEAD\n", "electric_ray\n", "sting Ray"]


def reference_nodes(ref_root):
    tree = ast.parse(open(os.path.join(ref_root, REL)).read())
    assigns = {t.id: n for n in tree.body if isinstance(n, ast.Assign) for t in n.targets
               if isinstance(t, ast.Name)}
    funcs = {n.name: n for n in tree.body if isinstance(n, ast.FunctionDef)}
    return assigns, funcs


def run_nodes(nodes, ns):
    exec(compile(ast.Module(body=list(nodes), type_ignores=[]), REL, "exec"), ns)
    return ns


def main(ref_root):
    assigns, funcs = reference_nodes(ref_root)
    tables = run_nodes([assigns["ALEXNET_CE"]], {})
    alexnet = tables["ALEXNET_CE"]

    quota = {}
    for g in range(1, 9):
        seen = [[] for _ in range(g)]
        for thread in range(g):
            ns = {"FLAGS": types.SimpleNamespace(gpu_index=",".join(str(i) for i in range(g))),
                  "ALEXNET_CE": dict(alexnet), "OURS_CE": {}, "ABSOLUTE_CE": {},
                  "print": lambda *a, **k: None,
                  "show_corruption_error_by_distortion":
                      lambda name, ckpt, gpu_id, t=thread: seen[t].append(name) or 0.5}
            run_nodes([funcs["process"]], ns)["process"](thread, "ckpt")
        quota[str(g)] = seen

    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "labels.txt")
        with open(path, "w") as f:
            f.writelines(LABEL_LINES)
        ns = {"tf": types.SimpleNamespace(gfile=types.SimpleNamespace(GFile=open))}
        synsets2idx = run_nodes([funcs["get_synsets2idx"]], ns)["get_synsets2idx"](path)

    gold = {"alexnet_ce": [[k, v] for k, v in alexnet.items()], "quota": quota,
            "label_lines": LABEL_LINES, "synsets2idx": synsets2idx}
    json.dump(gold, open(OUT, "w"), sort_keys=True, indent=1)
    print("wrote", OUT)


if __name__ == "__main__":
    if len(sys.argv) != 2 or not os.path.isfile(os.path.join(sys.argv[1], REL)):
        sys.exit("usage: python tests/golden/make_robustness_golden.py REFERENCE_DIR\n"
                 "  REFERENCE_DIR: a checkout of clovaai/assembled-cnn (the directory holding mce/)")
    main(os.path.abspath(sys.argv[1]))
