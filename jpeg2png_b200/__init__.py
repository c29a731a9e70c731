"""jpeg2png_b200: the jpeg2png solver on H100.  `decode_jpeg` (jpeg2png_b200.decode) turns JPEG files
into CUDA tensors; torch is imported only when it is first used."""

__all__ = ['decode_jpeg']


def __getattr__(name):
    if name == 'decode_jpeg':
        from .decode import decode_jpeg
        return decode_jpeg
    raise AttributeError(f'module {__name__!r} has no attribute {name!r}')
