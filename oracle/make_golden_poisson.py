"""TEST INFRASTRUCTURE -- mints tests/golden/poisson.json from the UNMODIFIED reference scripts/exporter.py (ExportPoissonMesh) on CPU
(needs the reference source tree, see oracle/ref_import.py).

open3d, pymeshlab and the reference's Pipeline module are absent here, so the stubs of oracle/make_golden_pointcloud.py stand in.
Recorded: ExportPoissonMesh's fields and defaults, and what ``validate_pipeline`` does on a pipeline whose model lacks the normal output
(the lines it prints, with rich markup stripped, and its exit code) and on one that has it.

    python -m oracle.make_golden_poisson
"""
import dataclasses
import importlib.util
import json
import os
import re
import sys

import torch

from . import ref_import
from .make_golden_pointcloud import GOLDEN_DIR, install_stubs
from .make_golden_tsdf import describe_default


class _Console:
    def __init__(self):
        self.lines = []

    def print(self, *args, **kwargs):
        self.lines.append(re.sub(r"\[/?[a-z ]+\]", "", " ".join(str(a) for a in args)))


class _Pipeline:
    device = torch.device("cpu")

    def __init__(self, outputs):
        self.outputs = outputs
        self.bundles = []

    def model(self, ray_bundle):
        self.bundles.append(dict(origins=ray_bundle.origins.tolist(), directions=ray_bundle.directions.tolist()))
        return {k: torch.zeros(1, 3) for k in self.outputs}


def main():
    ref_import.install_shims()
    install_stubs({})
    spec = importlib.util.spec_from_file_location("ref_exporter_script", os.path.join(ref_import.REFERENCE_ROOT, "scripts", "exporter.py"))
    exporter = sys.modules[spec.name] = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(exporter)

    meta = {"fields": [[f.name, describe_default(f.default_factory() if f.default_factory is not dataclasses.MISSING else f.default)]
                       for f in dataclasses.fields(exporter.ExportPoissonMesh)], "validate_pipeline": {}}
    cases = {"missing_normals": (dict(), ("rgb", "depth", "normal")), "present": (dict(normal_output_name="normal"), ("rgb", "depth", "normal")),
             "open3d": (dict(normal_method="open3d"), ("rgb", "depth"))}
    for name, (kw, outputs) in cases.items():
        console = exporter.CONSOLE = _Console()
        cfg = exporter.ExportPoissonMesh(load_config=None, output_dir=None, **kw)
        pipe = _Pipeline(outputs)
        code = None
        try:
            cfg.validate_pipeline(pipe)
        except SystemExit as e:
            code = e.code
        meta["validate_pipeline"][name] = dict(kwargs=kw, outputs=list(outputs), printed=console.lines, exit_code=code, rays=pipe.bundles)
    print(json.dumps(meta["validate_pipeline"], indent=1))
    with open(os.path.join(GOLDEN_DIR, "poisson.json"), "w") as fh:
        json.dump(meta, fh, indent=1)


if __name__ == "__main__":
    main()
