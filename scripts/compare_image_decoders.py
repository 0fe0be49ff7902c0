"""Our PNG/JPEG decoders vs stb_image as run by the reference's own parser (oracle/_ref/libm2s_refloader.so)."""
import io, os, sys, tempfile
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import oracle
from util import write_image_glb
from mesh2splat_b200.gltf import load_glb
from PIL import Image

d = tempfile.mkdtemp(); rng = np.random.default_rng(5)
worst = 0
def cmp(blob, tag):
    global worst
    p = os.path.join(d, "t.glb"); write_image_glb(p, blob, "image/jpeg")
    ok, meshes = oracle.ref_load_glb(p)
    ours = load_glb(p).textures[0]
    t = meshes[0]["textures"].get(0)
    dd = np.abs(t.astype(int) - ours.astype(int))
    worst = max(worst, dd.max())
    if dd.max():
        print(tag, "max", dd.max(), "mean", round(dd.mean(), 4), "n", int((dd > 0).sum()))
for (w, h) in [(64, 48), (70, 37), (33, 65), (17, 9), (129, 95), (8, 8), (1, 1), (2, 3), (16, 16), (15, 17)]:
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.stack([128 + 100 * np.sin(xx / 9), 128 + 100 * np.cos(yy / 7), 128 + 60 * np.sin((xx + yy) / 11)], axis=-1)
    for noise in (0, 6, 60):
        im = np.clip(img + rng.normal(0, noise, img.shape), 0, 255).astype(np.uint8)
        for prog in (False, True):
            for ss in (0, 1, 2):
                for q in (30, 85, 100):
                    b = io.BytesIO(); Image.fromarray(im).save(b, "JPEG", quality=q, subsampling=ss, progressive=prog)
                    cmp(b.getvalue(), f"jpeg {w}x{h} noise{noise} prog{int(prog)} ss{ss} q{q}")
            b = io.BytesIO(); Image.fromarray(im[..., 0]).save(b, "JPEG", quality=85, progressive=prog); cmp(b.getvalue(), f"gray {w}x{h} prog{int(prog)}")
print("worst difference over all cases:", worst)
