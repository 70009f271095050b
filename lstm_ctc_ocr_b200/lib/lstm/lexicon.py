"""Lexicon files for lexicon-based reading (cfg.TEST.LEXICON): one word per line, UTF-8, blank lines skipped, surrounding
whitespace stripped.  Words are encoded with get_encode_decode_dict (cfg.CHARSET -> ids 1 .. len(CHARSET))."""
from .config import cfg, get_encode_decode_dict


def load_lexicon(path):
    """The words of `path` as id tuples, in file order (duplicates included; engine.Lexicon keeps the first).  A character outside
    cfg.CHARSET raises ValueError naming the file and line; so does a word longer than 63 characters."""
    enc, _ = get_encode_decode_dict()
    words = []
    with open(path, "r", encoding="utf-8") as f:
        for lineno, line in enumerate(f, 1):
            w = line.strip()
            if not w:
                continue
            bad = [ch for ch in w if ch not in enc or ch == cfg.SPACE_TOKEN]
            if bad:
                raise ValueError(f"{path}:{lineno}: {w!r} has a character outside cfg.CHARSET: {bad[0]!r}")
            if len(w) > 63:
                raise ValueError(f"{path}:{lineno}: {w!r} is longer than 63 characters")
            words.append(tuple(enc[ch] for ch in w))
    if not words:
        raise ValueError(f"{path}: no words")
    return words
