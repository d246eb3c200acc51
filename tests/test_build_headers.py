"""The incremental build (onnxstream_b200/build.py) rebuilds an object file when its source or a file of build.HEADERS is newer: every
header a source includes must be in that list, or an edit to it leaves stale objects behind."""
import os
import re

from onnxstream_b200 import build


def test_every_included_header_is_a_build_dependency():
    listed = {os.path.normpath(os.path.join(build.CSRC, h)) for h in build.HEADERS}
    missing = set()
    for name in sorted(os.listdir(build.CSRC)):
        if not name.endswith((".cu", ".cuh", ".cpp", ".h")):
            continue
        with open(os.path.join(build.CSRC, name)) as f:
            for inc in re.findall(r'^\s*#\s*include\s+"([^"]+)"', f.read(), re.M):
                path = os.path.normpath(os.path.join(build.CSRC, inc))
                if os.path.isfile(path) and path not in listed:
                    missing.add(f"{name}: {inc}")
    assert not missing, sorted(missing)
