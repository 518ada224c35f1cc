"""8-bit PNG files of the working directory: the encoder the GPU stages write their PNGs with (one IDAT, filter type 0, zlib level 1 by
default, encoded on the callers' thread pools) and a header reader that checks what a frame holds before it is decoded."""
import struct
import time
import zlib

import numpy as np

SIGNATURE = b"\x89PNG\r\n\x1a\n"


def _png_bytes(img, color_type, level):
    """An 8-bit PNG of img [h, w] or [h, w, 3] u8 (filter type 0 on every row, one zlib IDAT)."""
    h, w = img.shape[:2]
    raw = np.zeros((h, img[0].size + 1), np.uint8)
    raw[:, 1:] = img.reshape(h, -1)

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xffffffff)
    return (SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, color_type, 0, 0, 0)) +
            chunk(b"IDAT", zlib.compress(raw.tobytes(), level)) + chunk(b"IEND", b""))


def png_gray_bytes(img, level=1):
    """An 8-bit grayscale PNG of img [h, w] u8 (filter type 0 on every row, one zlib IDAT)."""
    img = np.ascontiguousarray(img, np.uint8)
    if img.ndim != 2:
        raise ValueError(f"a grayscale PNG needs an [h, w] image, not {img.shape}")
    return _png_bytes(img, 0, level)


def png_rgb_bytes(img, level=1):
    """An 8-bit RGB PNG (colour type 2) of img [h, w, 3] u8, whose channels are in PNG (R, G, B) order."""
    img = np.ascontiguousarray(img, np.uint8)
    if img.ndim != 3 or img.shape[2] != 3:
        raise ValueError(f"an RGB PNG needs an [h, w, 3] image, not {img.shape}")
    return _png_bytes(img, 2, level)


def write_png(fn, img):
    """Writes img ([h, w]: grayscale, [h, w, 3]: R, G, B) as fn; returns the seconds spent encoding and writing."""
    t = time.perf_counter()
    data = png_gray_bytes(img) if img.ndim == 2 else png_rgb_bytes(img)
    with open(fn, "wb") as f:
        f.write(data)
    return time.perf_counter() - t


def png_header(fn):
    """{"height", "width", "bit_depth", "color_type", "interlace", "exif"} of a PNG file, from its IHDR and a walk over its chunk
    headers (exif: an eXIf chunk is present).  Reads a few bytes per chunk, not the image data.  Raises ValueError for a file that is
    not a PNG or ends before its IEND chunk."""
    with open(fn, "rb", buffering=0) as f:
        head = f.read(33)
        if len(head) < 33 or head[:8] != SIGNATURE or head[12:16] != b"IHDR":
            raise ValueError(f"{fn}: not a PNG file")
        w, h, depth, ctype, _, _, interlace = struct.unpack(">IIBBBBB", head[16:29])
        out = {"height": h, "width": w, "bit_depth": depth, "color_type": ctype, "interlace": interlace, "exif": False}
        pos = 33
        while True:
            f.seek(pos)
            c = f.read(8)
            if len(c) < 8:
                raise ValueError(f"{fn}: truncated PNG file (no IEND chunk)")
            n, typ = struct.unpack(">I4s", c)
            if typ == b"eXIf":
                out["exif"] = True
            elif typ == b"IEND":
                return out
            pos += 12 + n
