"""Writes the deflate-encoder fixtures from the reference's own test data (run once; the outputs are committed):
  flate_block_tokens.json   the token lists of writeBlockTests (flate/huffman_bit_writer_test.go:108-163) as
                            {"input", "want", "wantNoInput", "tokens"}: file names as in the reference (testdata/...,
                            found in flate_testdata.zip under flate/), tokens as integers
  deflate_fuzz_corpus.zip   flate/testdata/fuzz/encode-raw-corpus.zip, every entry (each the raw fuzz input)
usage: make_deflate_fixtures.py REFERENCE_ROOT"""
import io
import json
import os
import re
import sys
import zipfile

HERE = os.path.dirname(os.path.abspath(__file__))


def block_tests(src):
    body = src[src.index("var writeBlockTests"):src.index("func TestWriteBlock(")]
    consts = {"ml": int(re.search(r"const ml = (0x[0-9a-fA-F]+)", src).group(1), 16)}
    out = []
    for m in re.finditer(r"\{\s*((?:input|want|wantNoInput|tokens):.*?)\n\t\},", body, re.S):
        item = m.group(1)
        t = {k: v for k, v in re.findall(r'(input|want|wantNoInput):\s*"([^"]*)"', item)}
        toks = re.search(r"tokens:\s*\[\]token\{([^}]*)\}", item).group(1)
        t["tokens"] = [consts[x] if x in consts else int(x, 0) for x in (y.strip() for y in toks.split(",")) if x]
        out.append({k: t.get(k, "") for k in ("input", "want", "wantNoInput")} | {"tokens": t["tokens"]})
    return out


def main(ref):
    src = open(os.path.join(ref, "flate", "huffman_bit_writer_test.go")).read()
    tests = block_tests(src)
    assert len(tests) == 9, len(tests)
    with open(os.path.join(HERE, "flate_block_tokens.json"), "w") as f:
        json.dump(tests, f, separators=(",", ":"))
    zin = zipfile.ZipFile(os.path.join(ref, "flate", "testdata", "fuzz", "encode-raw-corpus.zip"))
    pick = sorted(zin.namelist())
    with zipfile.ZipFile(os.path.join(HERE, "deflate_fuzz_corpus.zip"), "w", zipfile.ZIP_DEFLATED) as z:
        for n in pick:
            z.writestr(n, zin.read(n))
    print(len(tests), "block tests;", len(pick), "fuzz inputs")


if __name__ == "__main__":
    main(sys.argv[1])
