#!/usr/bin/env python
"""Word count over UTF-8 text on the GPU (examples/wc.py shape; dpark_b200/textingest.py reduce_tokens_utf8).

A seeded mixed Chinese/English corpus -- lines of 10 tokens drawn with Zipf(1.0) frequencies from 25 k English-like
and 25 k Chinese words of 1 to 4 characters, separated by ' ', U+3000 (ideographic space) or a tab -- is counted three
ways, each after a warm-up run of the same job:

  utf8     the device path: the ASCII pass declines, dpk_tokenize_utf8 tokenises, the GPU shuffle combines;
  rowwise  engine.TEXT_INGEST = False: the user's Python generator tokenises every line (the reference's way);
  ascii    the ASCII device path on an ASCII corpus with the same token ids and count.

The time is `reduceByKey(...)._materialize()` (ingest + tokenise + shuffle + the distinct words back on the host),
the median of --repeats runs.  Then, from the library's per-launch CUDA events (dpk_prof_*), the kernel times of
k_tok8_count / k_tok8_emit over the whole corpus against the algorithmic bytes (two passes over the text, the token
bytes the emit walks again and its 16 B of (start, length) per token), and k_tok_count / k_tok_emit on the ASCII
corpus; and the dispatch cost: reduce_tokens declining on the UTF-8 corpus (its copy to the device, the ASCII count
pass and one host read) before reduce_tokens_utf8 starts from the beginning.  Word counts of the three ways are
checked equal (utf8 against rowwise; ascii against a Counter).  Prints one JSON line last.

    python scripts/wc_utf8_e2e.py [--tokens 10000000] [--repeats 3] [--no-rowwise]
"""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def corpora(tokens, seed=1):
    rng = np.random.default_rng(seed)
    vocab_n = 50_000
    letters = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", dtype=np.uint8)
    english = ["".join(chr(c) for c in letters[rng.integers(0, 26, int(rng.integers(2, 10)))]) for _ in range(vocab_n // 2)]
    chinese = ["".join(chr(int(c)) for c in rng.integers(0x4E00, 0x9FA6, int(rng.integers(1, 5)))) for _ in range(vocab_n // 2)]
    vocab = [w for pair in zip(english, chinese) for w in pair]          # frequent ranks alternate the two languages
    w = 1.0 / np.arange(1, vocab_n + 1)
    lines_n = tokens // 10
    ids = np.searchsorted(np.cumsum(w / w.sum()), rng.random(lines_n * 10)).reshape(lines_n, 10)
    seps = [" ", "\u3000", "\t"]
    sep_of = rng.choice(3, lines_n, p=[0.6, 0.3, 0.1])
    utf8 = "".join(seps[s].join(vocab[i] for i in row) + "\n" for row, s in zip(ids.tolist(), sep_of.tolist()))
    ascii_ = "".join(" ".join("w%d" % i for i in row) + "\n" for row in ids.tolist())
    return utf8.encode("utf-8"), ascii_.encode("ascii"), lines_n * 10


def fm(x):
    for wd in x.strip().split():
        yield (wd, 1)


def gpu_conditions():
    import torch
    q = "name,power.limit,clocks.max.sm"
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the numbers still stand; say what could not be read
        smi = "nvidia-smi unavailable (%s)" % type(e).__name__
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q + ": " + smi}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=10_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--no-rowwise", action="store_true")
    args = ap.parse_args()
    sys.argv = sys.argv[:1]
    import torch
    from dpark_b200 import DparkContext, engine, textingest
    from dpark_b200 import _native as nv
    if not torch.cuda.is_available():
        raise SystemExit("wc_utf8_e2e.py measures the GPU path: no CUDA device")
    torch.zeros(1, device="cuda")
    nv.lib()
    tmp = tempfile.mkdtemp(prefix="dpk_wc8_")
    t0 = time.perf_counter()
    utf8, ascii_, ntok = corpora(args.tokens)
    paths = {}
    for name, body in (("utf8", utf8), ("ascii", ascii_)):
        paths[name] = os.path.join(tmp, name + ".txt")
        with open(paths[name], "wb") as f:
            f.write(body)
    print("corpora: %d tokens each; UTF-8 %d bytes, ASCII %d bytes (%.1f s to generate)"
          % (ntok, len(utf8), len(ascii_), time.perf_counter() - t0))
    dc = DparkContext("local")

    spread = {}

    def job(path):
        sh = dc.textFile(path, numSplits=4).flatMap(fm).reduceByKey(lambda x, y: x + y, numSplits=6)
        torch.cuda.synchronize()
        a = time.perf_counter()
        sh._materialize()
        torch.cuda.synchronize()
        b = time.perf_counter()
        return b - a, sh

    def timed(path, repeats):
        job(path)                                   # warm-up: modules loaded, allocator grown
        runs = [job(path) for _ in range(repeats)]
        spread[path] = [round(t, 4) for t, _ in runs]
        return statistics.median(t for t, _ in runs), runs[-1][1]

    res = {"tokens": ntok, "utf8_bytes": len(utf8), "ascii_bytes": len(ascii_)}
    res.update(gpu_conditions())
    calls = []
    for name in ("reduce_tokens", "reduce_tokens_utf8"):
        real = getattr(textingest, name)
        setattr(textingest, name, lambda *a, _r=real, _n=name, **kw: calls.append(_n) or _r(*a, **kw))
    t_utf8, sh = timed(paths["utf8"], args.repeats)
    assert calls[-2:] == ["reduce_tokens", "reduce_tokens_utf8"], calls
    got = dict(sh.collect())
    t_ascii, sh_a = timed(paths["ascii"], args.repeats)
    assert calls[-1] == "reduce_tokens"
    want_a = collections.Counter(ascii_.decode("ascii").split())
    assert dict(sh_a.collect()) == dict(want_a), "ASCII word counts differ"
    res.update(utf8_device_s=t_utf8, ascii_device_s=t_ascii, distinct_words=len(got),
               utf8_runs_s=spread[paths["utf8"]], ascii_runs_s=spread[paths["ascii"]])
    print("utf8 device path:  %.3f s (%.2e tokens/s), %d distinct words" % (t_utf8, ntok / t_utf8, len(got)))
    print("ascii device path: %.3f s (%.2e tokens/s) on the ASCII corpus" % (t_ascii, ntok / t_ascii))
    if not args.no_rowwise:
        engine.TEXT_INGEST = False
        sh_r = dc.textFile(paths["utf8"], numSplits=4).flatMap(fm).reduceByKey(lambda x, y: x + y, numSplits=6)
        a = time.perf_counter()
        sh_r._materialize()
        torch.cuda.synchronize()
        t_row = time.perf_counter() - a
        engine.TEXT_INGEST = True
        assert dict(sh_r.collect()) == got, "UTF-8 word counts differ between the device and the row-wise path"
        res["rowwise_s"] = t_row
        print("row-wise path:     %.3f s (%.2e tokens/s), one run; counts identical to the device path"
              % (t_row, ntok / t_row))

    # kernel times over the whole corpus, from the library's per-launch CUDA events
    def kernels(body, tokenize, labels, iters=10):
        d = torch.from_numpy(np.frombuffer(body, dtype=np.uint8).copy()).cuda()
        starts, lens, ok = tokenize(d)
        assert ok
        torch.cuda.synchronize()
        nv.prof_enable(True)
        for _ in range(iters):
            tokenize(d)
        torch.cuda.synchronize()
        rows = nv.prof_collect()
        nv.prof_enable(False)
        ms = {lab: statistics.median(t for n, t in rows if n == lab) for lab in labels}
        res["%s_kernel_ms_min_max" % tokenize.__name__] = {lab: [min(t for n, t in rows if n == lab),
                                                                max(t for n, t in rows if n == lab)] for lab in labels}
        return ms, int(starts.numel()), int(lens.sum().item())

    ms8, n8, tokb8 = kernels(utf8, nv.tokenize_utf8, ("tok8_count", "tok8_emit"))
    ms1, n1, tokb1 = kernels(ascii_, nv.tokenize, ("tok_count", "tok_emit"))
    assert n8 == n1 == ntok
    for tag, ms, body, n, tokb in (("utf8", ms8, utf8, n8, tokb8), ("ascii", ms1, ascii_, n1, tokb1)):
        algo = 2 * len(body) + tokb + 16 * n
        k = sum(ms.values())
        res["%s_kernel_ms" % tag] = ms
        res["%s_algorithmic_bytes" % tag] = algo
        res["%s_algorithmic_GBps" % tag] = algo / (k * 1e-3) / 1e9
        print("%s tokeniser kernels: %s, %.3f ms together; %d algorithmic bytes -> %.0f GB/s"
              % (tag, ", ".join("%s %.3f ms" % kv for kv in ms.items()), k, algo, algo / (k * 1e-3) / 1e9))

    # dispatch cost: the ASCII pass declining on the UTF-8 corpus before the UTF-8 pass starts over
    from dpark_b200.engine import ShuffleResult
    tf = dc.textFile(paths["utf8"], numSplits=4)
    rdd = tf.flatMap(fm).reduceByKey(lambda x, y: x + y, numSplits=6)
    dev = torch.device("cuda", torch.cuda.current_device())
    part = rdd.partitioner
    decl = []
    for _ in range(args.repeats + 1):
        torch.cuda.synchronize()
        a = time.perf_counter()
        r = textingest.reduce_tokens(tf, range(len(tf.splits)), 6, part.thresholds, rdd.op, dev, ShuffleResult(6))
        torch.cuda.synchronize()
        decl.append(time.perf_counter() - a)
        assert r is None
    t_decl = statistics.median(decl[1:])
    res["dispatch_decline_s"] = t_decl
    res["dispatch_decline_runs_s"] = [round(t, 4) for t in decl[1:]]
    print("dispatch: reduce_tokens declines on the UTF-8 corpus in %.3f s = %.1f%% of the UTF-8 job"
          % (t_decl, 100 * t_decl / t_utf8))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
