"""What the UTF-8 tokeniser tests share: Python's own whitespace set, seeded mixed-language text, and the byte strings
that probe strict UTF-8 decoding."""
import numpy as np

# every code point str.split() / str.strip() without arguments splits on, taken from Python itself
WHITESPACE = [c for c in range(0x110000) if chr(c).isspace()]
NON_SURROGATES = [c for c in range(0x110000) if not 0xD800 <= c <= 0xDFFF]

_LATIN1 = [chr(c) for c in range(0xA1, 0x100) if not chr(c).isspace()]
_CJK = [chr(c) for c in range(0x4E00, 0xA000)]
_EMOJI = [chr(c) for c in range(0x1F300, 0x1F650)]
_CYRILLIC = [chr(c) for c in range(0x410, 0x450)]
_NOT_WS = ["\ufeff", "\u200b", "\u180e", "\x00", "\x7f", "\U0010ffff"]    # look like separators, are not whitespace


def random_text(seed, nchars, ascii_only=False):
    """Seeded text of about `nchars` characters: words of ASCII, Latin-1, Cyrillic, CJK and emoji letters (or ASCII
    only), separated by one or more of Python's whitespace characters, with a BOM, U+200B and U+180E inside words."""
    rng = np.random.default_rng(seed)
    ascii_letters = [chr(c) for c in range(0x21, 0x7F)]
    alphabets = [ascii_letters] if ascii_only else [ascii_letters, _LATIN1, _CYRILLIC, _CJK, _EMOJI, _NOT_WS]
    seps = [" ", "\t", "\n"] if ascii_only else [chr(c) for c in WHITESPACE]
    out, n = [], 0
    while n < nchars:
        alpha = alphabets[int(rng.integers(0, len(alphabets)))]
        word = "".join(alpha[int(i)] for i in rng.integers(0, len(alpha), int(rng.integers(1, 9))))
        sep = "".join(seps[int(i)] for i in rng.integers(0, len(seps), int(rng.integers(1, 3))))
        out.append(word + sep)
        n += len(word) + len(sep)
    return "".join(out)


def probe_sequences():
    """Byte strings that cover strict UTF-8 at the first, second, third and fourth byte: every 1- and 2-byte string;
    every lead E0..EF and F0..F4 with every second byte and valid, invalid and missing third (and fourth) bytes."""
    out = [bytes([a]) for a in range(256)] + [bytes([a, b]) for a in range(256) for b in range(256)]
    for a in range(0xE0, 0xF0):
        for b in range(256):
            out += [bytes([a, b, c]) for c in (0x80, 0x9F, 0xA0, 0xBF, 0x7F, 0xC0, 0x20)]
    for a in range(0xF0, 0xF5):
        for b in range(256):
            for c in (0x80, 0xBF, 0x7F, 0xC0):
                out += [bytes([a, b, c])] + [bytes([a, b, c, d]) for d in (0x80, 0xBF, 0x7F, 0xC0, 0x20)]
    return out


def decodes(b):
    try:
        return b.decode("utf-8")
    except UnicodeDecodeError:
        return None
