"""Writes tests/golden/eval_flags.json from the reference's evaluation CLI source (LADI_REFERENCE = a checkout of the reference): every
`parser.add_argument(...)` of src/eval.py as (flags, type, default, required, choices, action), read from the AST as
make_cli_golden.py does for src/inference.py (the module cannot be imported here: diffusers / accelerate are not installed), plus the
checkpoint-name prefixes its `latest` discovery filters on.

    python tests/golden/make_eval_golden.py
"""
import ast
import json
import os

SRC = os.path.join(os.environ["LADI_REFERENCE"], "src", "eval.py")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "eval_flags.json")


def main():
    tree = ast.parse(open(SRC).read())
    flags, prefixes = [], []
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "add_argument":
            names = [ast.literal_eval(a) for a in node.args]
            kw = {}
            for k in node.keywords:
                if k.arg == "help":
                    continue
                kw[k.arg] = k.value.id if isinstance(k.value, ast.Name) else ast.literal_eval(k.value)
            flags.append(dict(flags=names, line=node.lineno, **kw))
        # dirs = [d for d in dirs if d.startswith("<prefix>")]
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "startswith" and node.args:
            prefixes.append((node.lineno, ast.literal_eval(node.args[0])))
    flags.sort(key=lambda f: f["line"])
    json.dump(dict(source="src/eval.py", flags=flags, latest_prefixes=[p for _, p in sorted(prefixes)]), open(OUT, "w"), indent=1)
    print(f"{len(flags)} flags -> {OUT}")


if __name__ == "__main__":
    main()
