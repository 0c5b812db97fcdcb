"""The documentation stays truthful: every `alpa.<name>` / `global_config.<name>` it mentions exists, every repo path it
cites exists, and the quick-start tutorial's code runs as written."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DOCS = sorted(glob.glob(os.path.join(ROOT, "docs", "**", "*.md"), recursive=True)) + \
    [os.path.join(ROOT, n) for n in ("README.md", "DESIGN.md")]


def test_documented_api_names_exist():
    import alpa_b200 as alpa
    from alpa_b200.global_env import global_config
    missing = []
    for path in DOCS:
        text = open(path).read()
        for name in set(re.findall(r"\balpa\.([A-Za-z_][A-Za-z0-9_]*)", text)):
            if name in ("projects", "py", "md"):        # "alpa-projects/alpa", file names
                continue
            if not hasattr(alpa, name):
                missing.append((os.path.relpath(path, ROOT), f"alpa.{name}"))
        for name in set(re.findall(r"\bglobal_config\.([a-z_][a-z0-9_]*)", text)):
            if not hasattr(global_config, name):
                missing.append((os.path.relpath(path, ROOT), f"global_config.{name}"))
    assert not missing, missing


def test_documented_repo_paths_exist():
    missing = []
    pat = re.compile(r"`((?:alpa_b200|benchmark|examples|scripts|tests|profiles|docs)/[A-Za-z0-9_./{},*-]+)`")
    for path in DOCS:
        text = open(path).read()
        # citations of the reference repository ("reference: `benchmark/alpa/...`", tables with a Reference column) are
        # paths of that repository: skip paragraphs / table rows that say so
        chunks = [c for c in re.split(r"\n\s*\n|\n(?=\|)", text) if "eference" not in c]
        for ref in set(r for c in chunks for r in pat.findall(c)):
            ref = ref.split(":")[0].rstrip(".,")
            if any(ch in ref for ch in "{}*"):
                continue
            cand = os.path.join(ROOT, ref)
            in_reference = ref.startswith(("benchmark/alpa/", "examples/llm_serving/benchmark/", "docs/gallery/"))
            if not (os.path.exists(cand) or glob.glob(cand + "*") or in_reference):
                missing.append((os.path.relpath(path, ROOT), ref))
    assert not missing, missing


def test_quickstart_tutorial_code_runs():
    import alpa_b200 as alpa
    src = open(os.path.join(ROOT, "docs", "tutorials", "quickstart.md")).read()
    code = "\n".join(re.findall(r"```python\n(.*?)```", src, re.S))
    try:
        exec(compile(code, "quickstart.md", "exec"), {"__name__": "__main__"})
    finally:
        alpa.shutdown()


def test_ddp_comparison_tutorial_code_runs():
    import alpa_b200 as alpa
    src = open(os.path.join(ROOT, "docs", "tutorials", "alpa_vs_ddp_fsdp.md")).read()
    blocks = re.findall(r"```python\n(.*?)```", src, re.S)
    try:
        exec(compile(blocks[0], "alpa_vs_ddp_fsdp.md", "exec"), {"__name__": "__main__"})
        ns = {"alpa": alpa}
        exec(compile(blocks[1], "alpa_vs_ddp_fsdp.md#2", "exec"), ns)       # the method constructors are valid
        assert isinstance(ns["method"], alpa.PipeshardParallel)
    finally:
        alpa.shutdown()
