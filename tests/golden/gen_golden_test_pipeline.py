"""Golden data for the test pipeline: `test_pipeline` and `img_norm_cfg` of the reference's three DOTA configs
(configs/dota/orientedrepoints_{r50,r101,swin_tiny}_demo.py), evaluated from the config source with `ast` (the config
files import nothing, but mmcv's Config loader is not installed), stored as JSON (tuples become lists).

    python tests/golden/gen_golden_test_pipeline.py     # needs /root/reference; writes tests/golden/test_pipelines.json
"""
import ast
import json
import os

REF = "/root/reference/configs/dota"
NAMES = ("orientedrepoints_r50_demo", "orientedrepoints_r101_demo", "orientedrepoints_swin_tiny_demo")


def extract(path):
    """module-level assignments of img_norm_cfg and test_pipeline, evaluated in order (test_pipeline refers to
    img_norm_cfg through **)"""
    tree = ast.parse(open(path).read(), path)
    ns = {"dict": dict}
    for node in tree.body:
        if isinstance(node, ast.Assign) and len(node.targets) == 1 and isinstance(node.targets[0], ast.Name) \
                and node.targets[0].id in ("img_norm_cfg", "test_pipeline"):
            ns[node.targets[0].id] = eval(compile(ast.Expression(node.value), path, "eval"), {"__builtins__": {}}, ns)
    return {"img_norm_cfg": ns["img_norm_cfg"], "test_pipeline": ns["test_pipeline"]}


def main():
    out = {n: extract(os.path.join(REF, n + ".py")) for n in NAMES}
    dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_pipelines.json")
    with open(dst, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", dst)


if __name__ == "__main__":
    main()
