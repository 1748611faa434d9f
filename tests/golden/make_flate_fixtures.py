"""Writes the inflate fixtures from the reference's own test data (run once; the outputs are committed):
  flate_testdata.zip   flate/testdata/*.golden, *.in, *.expect, *.expect-noinput; gzip/testdata/issue6550.gz, test.json;
                       a seeded sample (<= 64 KiB each) of the raw inputs of flate/testdata/regression.zip as regress/*
  flate_tables.json    the byte / expected-outcome tables of gzip/gunzip_test.go (gunzipTests), zlib/reader_test.go
                       (zlibTests), flate/flate_test.go (TestStreams) and flate/reader_test.go (TestNlitOutOfRange), as
                       {"table", "desc", "format", "stream" (hex), "want"}: want is the content (hex) or an error name
usage: make_flate_fixtures.py REFERENCE_ROOT"""
import codecs
import io
import json
import os
import random
import re
import sys
import zipfile

HERE = os.path.dirname(os.path.abspath(__file__))


def go_groups(body):
    """Top-level {...} groups of a Go composite literal body."""
    out, depth, start, i = [], 0, None, 0
    while i < len(body):
        c = body[i]
        if c == '"':
            j = i + 1
            while body[j] != '"':
                j += 2 if body[j] == "\\" else 1
            i = j
        elif c == "{":
            if depth == 0:
                start = i + 1
            depth += 1
        elif c == "}":
            depth -= 1
            if depth == 0:
                out.append(body[start:i])
        i += 1
    return out


def go_fields(group):
    """Top-level comma-separated fields of one struct literal."""
    out, depth, cur, i = [], 0, "", 0
    while i < len(group):
        c = group[i]
        if c == '"':
            j = i + 1
            while group[j] != '"':
                j += 2 if group[j] == "\\" else 1
            cur += group[i:j + 1]
            i = j + 1
            continue
        if c in "{(":
            depth += 1
        elif c in "})":
            depth -= 1
        if c == "," and depth == 0:
            out.append(cur.strip())
            cur = ""
        else:
            cur += c
        i += 1
    if cur.strip():
        out.append(cur.strip())
    return out


def go_value(f):
    f = f.strip()
    if f.startswith("[]byte{"):
        consts = {"gzipID1": 0x1f, "gzipID2": 0x8b, "gzipDeflate": 8}
        out = []
        for x in re.findall(r"0x[0-9a-fA-F]+|\d+|'.'|[A-Za-z_]\w*", f[len("[]byte{"):-1]):
            out.append(ord(x[1]) if x.startswith("'") else (consts[x] if x in consts else int(x, 0)))
        return bytes(out)
    if f.startswith('"'):
        parts = re.findall(r'"((?:[^"\\]|\\.)*)"', f)
        s = "".join(parts)
        return codecs.escape_decode(s.encode("utf-8"))[0]
    return f                                            # nil, io.EOF, ErrChecksum, ...


def strip_comments(src):
    return re.sub(r"//[^\n]*", "", src)


def table(path, name):
    src = strip_comments(open(path).read())
    m = re.search(r"var %s = \[\]\w+\{(.*?)\n\}\n" % name, src, re.S)
    return [[go_value(f) for f in go_fields(g)] for g in go_groups(m.group(1))]


def main(ref):
    rows = []
    for f in table(os.path.join(ref, "gzip/gunzip_test.go"), "gunzipTests"):
        name, desc, raw, gz, err = f
        rows.append({"table": "gunzipTests", "desc": desc.decode("utf-8"), "format": 2, "stream": gz.hex(),
                     "want": raw.hex() if err == "nil" else err})
    for f in table(os.path.join(ref, "zlib/reader_test.go"), "zlibTests"):
        desc, raw, comp, dct, err = f
        if dct != "nil":
            continue                                    # preset dictionaries: not offered
        rows.append({"table": "zlibTests", "desc": desc.decode("utf-8"), "format": 1, "stream": comp.hex(),
                     "want": raw.hex() if err == "nil" else err})
    src = strip_comments(open(os.path.join(ref, "flate/flate_test.go")).read())
    body = re.search(r"func TestStreams.*?\}\{(.*?)\n\t\}\}", src, re.S).group(1)
    for g in go_groups(body + "}"):
        desc, stream, want = [go_value(x) for x in go_fields(g)]
        rows.append({"table": "TestStreams", "desc": desc.decode(), "format": 0, "stream": stream.decode(),
                     "want": "fail" if want == b"fail" else want.decode()})
    nlit = re.search(r'func TestNlitOutOfRange.*?NewReader\(strings.NewReader\(\s*(".*?")\)\)\)', open(
        os.path.join(ref, "flate/reader_test.go")).read(), re.S).group(1)
    rows.append({"table": "TestNlitOutOfRange", "desc": "nlit = 288", "format": 0, "stream": go_value(nlit).hex(), "want": "fail"})
    with open(os.path.join(HERE, "flate_tables.json"), "w") as fo:
        json.dump(rows, fo, indent=0)
    zb = io.BytesIO()
    with zipfile.ZipFile(zb, "w", zipfile.ZIP_DEFLATED) as z:
        td = os.path.join(ref, "flate/testdata")
        for fn in sorted(os.listdir(td)):
            if fn.endswith((".golden", ".in", ".expect", ".expect-noinput")):
                z.write(os.path.join(td, fn), "flate/" + fn)
        for fn in ("issue6550.gz", "test.json"):
            z.write(os.path.join(ref, "gzip/testdata", fn), "gzip/" + fn)
        with zipfile.ZipFile(os.path.join(td, "regression.zip")) as rz:
            names = [n for n in sorted(rz.namelist()) if 0 < rz.getinfo(n).file_size <= 65536]
            for n in random.Random(1).sample(names, min(48, len(names))):
                z.writestr("regress/" + os.path.basename(n), rz.read(n))
    with open(os.path.join(HERE, "flate_testdata.zip"), "wb") as fo:
        fo.write(zb.getvalue())
    print(len(rows), "table rows")


if __name__ == "__main__":
    main(sys.argv[1])
