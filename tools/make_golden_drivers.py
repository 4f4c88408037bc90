"""Names the reference's driver scripts use, for tests/test_dropin_cpu.py: per script the modules it imports and
every unqualified name / first-level attribute it reads that the script does not define itself.

    python tools/make_golden_drivers.py     # needs the reference tree; writes tests/golden/driver_names.json
"""
import ast
import builtins
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("FPOSE_REFERENCE", "/root/reference")
# attribute owners that are the script's own objects (argparse results, readers, the estimator, open3d debug code)
LOCAL_OWNERS = {"run_demo.py": ("args", "parser", "o3d"),
                "run_linemod.py": ("opt", "parser", "o3d", "reader", "reader_tmp", "est"),
                "run_ycb_video.py": ("opt", "parser", "o3d", "reader", "reader_tmp", "est")}


def names(path, local_owners):
    tree = ast.parse(open(path).read())
    imports = [ast.unparse(n) for n in tree.body if isinstance(n, (ast.Import, ast.ImportFrom))]
    assigned, used, attrs = set(), set(), set()
    for node in ast.walk(tree):
        if isinstance(node, ast.Name):
            (assigned if isinstance(node.ctx, ast.Store) else used).add(node.id)
        elif isinstance(node, ast.Attribute) and isinstance(node.value, ast.Name):
            attrs.add((node.value.id, node.attr))
        elif isinstance(node, (ast.FunctionDef, ast.arg)):
            assigned.add(node.name if isinstance(node, ast.FunctionDef) else node.arg)
    need = sorted(n for n in used - assigned - set(dir(builtins)) if n != "__file__")
    mod_attrs = sorted([m, a] for (m, a) in attrs if m in need and m not in local_owners)
    return {"imports": imports, "names": need, "attributes": mod_attrs}


def main():
    out = {s: names(os.path.join(REF, s), owners) for s, owners in LOCAL_OWNERS.items()}
    path = os.path.join(ROOT, "tests", "golden", "driver_names.json")
    with open(path, "w") as fh:
        fh.write("{\n" + ",\n".join(f" {json.dumps(s)}: {json.dumps(out[s], sort_keys=True)}" for s in sorted(out)) + "\n}\n")
    print(path, {s: len(v["names"]) for s, v in out.items()})


if __name__ == "__main__":
    main()
