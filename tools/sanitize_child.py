"""Small solves through the C ABI for compute-sanitizer (tools/run_sanitizers.sh): every kernel family once
— joint 4:4:4, joint 4:2:0 with a frame larger than the luma grid, one-plane (-s) solves, odd sampling —
and four-component files through decode_jpeg (device entropy decoding and the four-plane export), and
CMYK encoding through the three JPEG encoders."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jpeg2png_b200 import synth  # noqa: E402
from tests import helpers as H  # noqa: E402

cases = [
    (136, 72, 50, '4:4:4', [0, 1, 2], 0.7, [0.001, 0.0, 0.01], 4),
    (200, 120, 30, '4:2:0', [0, 1, 2], 0.3, [0.001] * 3, 4),
    (256, 256, 10, '4:2:0', [1], 0.3, [0.001], 3),
    (64, 64, 90, '4:4:4', [0], 0.0, [0.0], 3),
]
for w, h, q, ss, channels, weight, pw, iters in cases:
    img = synth.synth_coefs(w, h, q, ss, seed=99 + w)
    f = H.decode_planes(img, channels)
    out = H.run_compute('product', img, channels, weight, pw, iters, f)
    print('ok', w, h, ss, channels, float(out[0].sum()))
img = synth.random_coefs([(40, 24), (24, 16), (16, 8)], [(1, 1), (2, 2), (3, 4)], 1)
out = H.run_compute('product', img, [0, 1, 2], 0.4, [0.001] * 3, 3, H.decode_planes(img))
print('ok random planes', float(out[0].sum()))

# four-component files (DESIGN §7q): the four-plane device entropy path (j2p_entropy_pack4) and
# j2p_session_export_four in its row and tiled mappings, CMYK and YCCK, four channels and RGB
import torch  # noqa: E402

from jpeg2png_b200 import decode_jpeg  # noqa: E402
from tests import cmyk_synth as S  # noqa: E402

four = [S.pillow_cmyk(61, 37, 75, seed=2), S.ycck_file(45, 35, [(2, 2), (1, 1), (1, 1), (2, 2)], 8, restart_interval=2)[0],
        S.ycck_file(53, 29, [(1, 1)] * 4, 13, transform=0, interleaved=False)[0]]
for mode, dtype in (('UNCHANGED', torch.uint8), ('UNCHANGED', torch.float32), ('RGB', torch.uint8)):
    for orient in (False, True):
        files = [f[:2] + S.exif_segment(6) + f[2:] for f in four] if orient else four
        ts = decode_jpeg(files, mode=mode, dtype=dtype, iterations=2, apply_exif_orientation=orient)
        torch.cuda.synchronize()
        print('ok four-component', mode, dtype, 'oriented' if orient else 'plain', [tuple(t.shape) for t in ts])

# CMYK encoding (DESIGN §7r): libj2pjpegenc.so, libj2pjpegopt.so and libj2pjpegprog.so on four-channel
# tensors, with and without restart intervals, strided and in two samplings
from jpeg2png_b200 import encode_jpeg  # noqa: E402
from tests import cmyk_jpeg_cases as K  # noqa: E402

xs = [torch.from_numpy(K.cmyk(kind, h, w, 3)).cuda() for kind, h, w in (('cartoon', 37, 53), ('noise', 16, 24), ('flat128', 1, 1))]
xs.append(xs[0].permute(2, 0, 1).contiguous().permute(1, 2, 0)[::2, 1:])
for mode in K.MODES.values():
    for s, kw in (('4:2:0', {}), ('4:4:4', {'restart_marker_rows': 1})):
        fs = encode_jpeg(xs, layout='HWC', subsampling=s, cmyk=True, **mode, **kw)
        torch.cuda.synchronize()
        print('ok cmyk encode', mode, s, kw, [len(f) for f in fs])
