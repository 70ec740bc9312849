"""benchmarks/harness.py without a GPU: the one JSON line on stdout, the fresh-process runner, and the rules that keep every
measuring decision in the harness (no script imports another; stdout diversion and device events only in the harness)."""
import ast
import glob
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BENCH = os.path.join(ROOT, "benchmarks")
SCRIPTS = sorted(glob.glob(os.path.join(BENCH, "*.py")))
NAMES = {os.path.splitext(os.path.basename(p))[0] for p in SCRIPTS}


def _child(code, tmp_path, name="child.py"):
    path = tmp_path / name
    path.write_text("import sys\nsys.path.insert(0, %r)\n" % BENCH + code)
    return str(path)


def test_emit_is_the_only_line_on_stdout(tmp_path):
    script = _child("import os\nimport harness\nharness.divert_stdout()\nprint('python noise')\n"
                    "os.write(1, b'fd noise\\n')\nharness.emit({'value': 1.5, 'gpu': {'name': 'x'}})\n", tmp_path)
    r = subprocess.run([sys.executable, script], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert r.stdout.splitlines() == [json.dumps({"value": 1.5, "gpu": {"name": "x"}})]
    assert "python noise" in r.stderr and "fd noise" in r.stderr


def test_in_fresh_process_returns_the_last_json_line(tmp_path):
    sys.path.insert(0, BENCH)
    import harness
    script = _child("print('{\"first\": 1}')\nprint('not json')\nprint('{\"last\": [2, 3]}')\n", tmp_path)
    assert harness.in_fresh_process(script, []) == {"last": [2, 3]}
    failing = _child("sys.stderr.write('early\\n' + 'x' * 3000 + 'the end of stderr\\n')\nsys.exit(3)\n", tmp_path, "failing.py")
    with pytest.raises(SystemExit) as e:
        harness.in_fresh_process(failing, ["--flag", "v"])
    assert "the end of stderr" in str(e.value) and "early" not in str(e.value)


def test_no_script_imports_another():
    for path in SCRIPTS:
        tree = ast.parse(open(path).read())
        for node in ast.walk(tree):
            if isinstance(node, ast.Import):
                mods = [a.name.split(".")[0] for a in node.names]
            elif isinstance(node, ast.ImportFrom):
                mods = [(node.module or "").split(".")[0]]
            else:
                continue
            for m in mods:
                assert m == "harness" or m not in NAMES, "%s imports benchmarks/%s.py" % (os.path.basename(path), m)


def test_plumbing_lives_only_in_the_harness():
    for path in SCRIPTS:
        if os.path.basename(path) == "harness.py":
            continue
        src = open(path).read()
        for needle in ("_REAL_STDOUT", "dup2", "torch.cuda.Event"):
            assert needle not in src, "%s has %s" % (os.path.basename(path), needle)


@pytest.mark.parametrize("path", [p for p in SCRIPTS if "argparse" in open(p).read()], ids=os.path.basename)
def test_help_exits_zero_without_a_gpu(path):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, path, "--help"], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "usage:" in r.stdout + r.stderr
