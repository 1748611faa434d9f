#!/usr/bin/env python3
"""Regenerates the LZ4 converter fixtures of tests/golden/ from the reference's test data (run where the reference is
mounted at /root/reference).  Data only, never source code:

  lz4_convert_corpus_raw.zip     s2/testdata/fuzz/lz4-convert-corpus-raw.zip: 108 raw LZ4 blocks (FuzzLZ4Block, s2/lz4convert_test.go:354)
  lz4_fuzz_block.zip             s2/testdata/fuzz/FuzzLZ4Block.zip: 244 seeds, turned from go-fuzz text form into raw bytes
"""
import ast
import os
import re
import shutil
import zipfile

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))


def gofuzz_bytes(text):
    """The []byte value of a go-fuzz corpus file ("go test fuzz v1" + one []byte(...) line, a Go string literal)."""
    line = text.decode("utf-8").split("\n")[1].strip()
    assert line.startswith("[]byte(") and line.endswith(")"), line
    lit = line[len("[]byte("):-1]
    if lit.startswith("`"):
        return lit[1:-1].encode("utf-8")
    # Go and Python agree on \xNN, \n, \t, \\, \" ...; raw UTF-8 text and \u / \U escapes become \x escapes first
    lit = re.sub(r"\\[uU]([0-9a-fA-F]{4,8})", lambda m: "".join("\\x%02x" % b for b in chr(int(m.group(1), 16)).encode("utf-8")), lit)
    lit = "".join(ch if ord(ch) < 128 else "".join("\\x%02x" % b for b in ch.encode("utf-8")) for ch in lit)
    return ast.literal_eval("b" + lit)


def main():
    shutil.copy(f"{REF}/s2/testdata/fuzz/lz4-convert-corpus-raw.zip", f"{HERE}/lz4_convert_corpus_raw.zip")
    os.chmod(f"{HERE}/lz4_convert_corpus_raw.zip", 0o644)
    src = zipfile.ZipFile(f"{REF}/s2/testdata/fuzz/FuzzLZ4Block.zip")
    out = zipfile.ZipFile(f"{HERE}/lz4_fuzz_block.zip", "w", zipfile.ZIP_DEFLATED, compresslevel=9)
    for info in sorted(src.infolist(), key=lambda i: i.filename):
        if info.is_dir():
            continue
        zi = zipfile.ZipInfo(info.filename, date_time=(2020, 1, 1, 0, 0, 0))     # fixed stamp: the file is reproducible
        zi.compress_type = zipfile.ZIP_DEFLATED
        out.writestr(zi, gofuzz_bytes(src.read(info)))
    out.close()


if __name__ == "__main__":
    main()
