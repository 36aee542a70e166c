"""Writes tests/golden/metrics_flags.json from the reference's metric script source (LADI_REFERENCE = a checkout of the reference): every
`parser.add_argument(...)` of src/utils/val_metrics.py as (flags, type, default, required, choices, action), read from the AST as
make_eval_golden.py does for src/eval.py (the module cannot be imported here: cleanfid / torchmetrics are not installed).

    python tests/golden/make_metrics_golden.py
"""
import ast
import json
import os

SRC = os.path.join(os.environ["LADI_REFERENCE"], "src", "utils", "val_metrics.py")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "metrics_flags.json")


def main():
    tree = ast.parse(open(SRC).read())
    flags = []
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "add_argument":
            names = [ast.literal_eval(a) for a in node.args]
            kw = {}
            for k in node.keywords:
                if k.arg == "help":
                    continue
                kw[k.arg] = k.value.id if isinstance(k.value, ast.Name) else ast.literal_eval(k.value)
            flags.append(dict(flags=names, line=node.lineno, **kw))
    flags.sort(key=lambda f: f["line"])
    json.dump(dict(source="src/utils/val_metrics.py", flags=flags), open(OUT, "w"), indent=1)
    print(f"{len(flags)} flags -> {OUT}")


if __name__ == "__main__":
    main()
