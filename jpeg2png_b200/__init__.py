"""jpeg2png_b200: the jpeg2png solver on H100.  `decode_jpeg` (jpeg2png_b200.decode) turns JPEG files
into CUDA tensors (RGB, or one channel for grayscale files and `mode='GRAY'`), `encode_png`
(jpeg2png_b200.encode, RGB or gray) and `encode_jpeg` (jpeg2png_b200.jpeg_encode, RGB or gray,
and with `cmyk=True` four-channel CMYK tensors as Pillow's Adobe CMYK files) turn such tensors into PNG or JPEG files on the device (`encode_jpeg(..., optimize=True)` with
per-image optimized Huffman tables, as Pillow's `optimize=True`, and `encode_jpeg(...,
progressive=True)` with Pillow's progressive files, and `encode_jpeg(..., qtables=)` with given
quantisation tables, per image if need be); `keep_settings` reads a JPEG file's tables and
sampling, as Pillow's quality='keep' re-uses them; `write_objective_csv` writes the objective logs of
`decode_jpeg(..., return_objective=True)` as the command line's -c file; torch is imported only when
one of them is first used."""

__all__ = ['decode_jpeg', 'encode_png', 'encode_jpeg', 'keep_settings', 'write_objective_csv']


def __getattr__(name):
    if name == 'decode_jpeg':
        from .decode import decode_jpeg
        return decode_jpeg
    if name == 'write_objective_csv':
        from .decode import write_objective_csv
        return write_objective_csv
    if name == 'encode_png':
        from .encode import encode_png
        return encode_png
    if name == 'encode_jpeg':
        from .jpeg_encode import encode_jpeg
        return encode_jpeg
    if name == 'keep_settings':
        from .jpeg_encode import keep_settings
        return keep_settings
    raise AttributeError(f'module {__name__!r} has no attribute {name!r}')
