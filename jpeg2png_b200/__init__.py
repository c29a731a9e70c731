"""jpeg2png_b200: the jpeg2png solver on H100.  `decode_jpeg` (jpeg2png_b200.decode) turns JPEG files
into CUDA tensors, `encode_png` (jpeg2png_b200.encode) turns such tensors into PNG files on the
device; torch is imported only when one of them is first used."""

__all__ = ['decode_jpeg', 'encode_png']


def __getattr__(name):
    if name == 'decode_jpeg':
        from .decode import decode_jpeg
        return decode_jpeg
    if name == 'encode_png':
        from .encode import encode_png
        return encode_png
    raise AttributeError(f'module {__name__!r} has no attribute {name!r}')
