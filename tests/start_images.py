"""The scanners of tests/golden/start_images.json.xz (written by tests/golden/make_start_images.py): per pattern set the
forward glued HalfFinalScanner image, the glued reversed image and one reversed image per regexp.  Nothing under
pire_b200/ imports it."""
import base64
import json
import lzma
import os

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "golden", "start_images.json.xz")


def _unpack(b64):
    return lzma.decompress(base64.b64decode(b64))


def load_start_images():
    with open(PATH, "rb") as f:
        raw = json.loads(lzma.decompress(f.read()))
    return {name: {"patterns": [(p.encode("latin-1"), o) for p, o in e["patterns"]], "forward": _unpack(e["forward"]),
                   "reversed": _unpack(e["reversed"]), "per_regexp": [_unpack(x) for x in e["per_regexp"]]}
            for name, e in raw.items()}


START_IMAGES = load_start_images()
