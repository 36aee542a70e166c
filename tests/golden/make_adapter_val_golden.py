"""Writes tests/golden/adapter_val_flags.json from the reference's inversion-adapter trainer and its validation function
(LADI_REFERENCE = a checkout of the reference), read from the AST as make_cli_golden.py does (the modules cannot be imported here:
diffusers / accelerate are not installed):
  * every `parser.add_argument(...)` of src/train_inversion_adapter.py as (flags, type, default, required, choices, action);
  * the dataset `outputlist` it validates with, and the flag that appends 'clip_cloth_features' to it;
  * the `save_name=` it passes to `generate_images_inversion_adapter` (an f-string over the global step), kept as its format string;
  * of `generate_images_inversion_adapter` (src/utils/image_from_pipe.py): the parameter names, their defaults and the `category_text`
    dict of its prompt template.

    python tests/golden/make_adapter_val_golden.py
"""
import ast
import json
import os

REF = os.environ["LADI_REFERENCE"]
TRAIN = os.path.join(REF, "src", "train_inversion_adapter.py")
FROM_PIPE = os.path.join(REF, "src", "utils", "image_from_pipe.py")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "adapter_val_flags.json")


def _fstring(node):
    """An f-string as its format string: f'imgs_step_{global_step}' -> 'imgs_step_{global_step}'."""
    return "".join(v.value if isinstance(v, ast.Constant) else "{" + ast.unparse(v.value) + "}" for v in node.values)


def _trainer():
    tree = ast.parse(open(TRAIN).read())
    flags, outputlist, clip_flag, save_name = [], None, None, None
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "add_argument":
            kw = {k.arg: (k.value.id if isinstance(k.value, ast.Name) else ast.literal_eval(k.value)) for k in node.keywords if k.arg != "help"}
            flags.append(dict(flags=[ast.literal_eval(a) for a in node.args], line=node.lineno, **kw))
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "outputlist" for t in node.targets):
            outputlist = ast.literal_eval(node.value)
        # if args.<flag>: outputlist.append('clip_cloth_features')
        if isinstance(node, ast.If) and isinstance(node.test, ast.Attribute):
            for st in node.body:
                c = getattr(st, "value", None)
                if (isinstance(c, ast.Call) and isinstance(c.func, ast.Attribute) and c.func.attr == "append"
                        and isinstance(c.func.value, ast.Name) and c.func.value.id == "outputlist"):
                    clip_flag = dict(flag="--" + node.test.attr, appends=ast.literal_eval(c.args[0]))
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == "generate_images_inversion_adapter":
            for k in node.keywords:
                if k.arg == "save_name":
                    save_name = _fstring(k.value)
    flags.sort(key=lambda f: f["line"])
    return flags, outputlist, clip_flag, save_name


def _validation_function():
    tree = ast.parse(open(FROM_PIPE).read())
    fn = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == "generate_images_inversion_adapter")
    names = [a.arg for a in fn.args.args]
    defaults = dict(zip(names[len(names) - len(fn.args.defaults):], [ast.literal_eval(d) for d in fn.args.defaults]))
    category_text = next(ast.literal_eval(n.value) for n in ast.walk(fn)
                         if isinstance(n, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "category_text" for t in n.targets))
    return names, defaults, category_text


def main():
    flags, outputlist, clip_flag, save_name = _trainer()
    params, defaults, category_text = _validation_function()
    json.dump(dict(source=["src/train_inversion_adapter.py", "src/utils/image_from_pipe.py"], flags=flags, outputlist=outputlist,
                   outputlist_append=clip_flag, save_name=save_name, function_params=params, function_defaults=defaults,
                   category_text=category_text), open(OUT, "w"), indent=1)
    print(f"{len(flags)} flags -> {OUT}")


if __name__ == "__main__":
    main()
