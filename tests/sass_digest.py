"""Per-function digest of a cubin / object's SASS (cuobjdump -sass), with addresses and encodings stripped: two builds of the same kernels compare
equal iff every function has the same instruction sequence."""
from __future__ import annotations

import hashlib
import re
import subprocess

_ADDR = re.compile(r"/\*[0-9a-f]{4,}\*/")
_ENC = re.compile(r"/\* 0x[0-9a-f]+ \*/")


def sass_digests(obj_path: str, cuobjdump: str = "cuobjdump") -> dict:
    text = subprocess.run([cuobjdump, "-sass", obj_path], check=True, capture_output=True, text=True).stdout
    out, name, body = {}, None, []
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                out[name] = hashlib.sha256("\n".join(body).encode()).hexdigest()
            name, body = m.group(1), []
            continue
        if name:
            s = _ENC.sub("", _ADDR.sub("", line)).strip()
            if s:
                body.append(s)
    if name:
        out[name] = hashlib.sha256("\n".join(body).encode()).hexdigest()
    return out
