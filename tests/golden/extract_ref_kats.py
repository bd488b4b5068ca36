#!/usr/bin/env python3
"""Extract the reference's golden vectors for the HashJoin / HashAgg / dispatch path into JSON.

Reads a checkout of risingwavelabs/risingwave; the tests only read the committed JSON:

    python tests/golden/extract_ref_kats.py <risingwave checkout> [output directory, default: this directory]

Outputs (committed):
    tests/golden/hash_join_kats.json   <- src/stream/src/executor/hash_join.rs  #[tokio::test]s
    tests/golden/hash_agg_kats.json    <- src/stream/tests/integration_tests/hash_agg.rs
    tests/golden/agg_func_kats.json    <- src/expr/impl/src/aggregate/general.rs tests
    tests/golden/filter_kats.json      <- src/stream/src/executor/filter.rs tests
    tests/golden/nexmark_q4_fixture.json <- e2e_test/nexmark/insert_{auction,bid}.slt.part + e2e_test/streaming/nexmark/q4.slt.part
    tests/golden/nexmark_q7_fixture.json <- e2e_test/nexmark/insert_bid.slt.part + e2e_test/streaming/nexmark/q7.slt.part
    tests/golden/nexmark_q8_fixture.json <- e2e_test/nexmark/insert_{person,auction}.slt.part + e2e_test/streaming/nexmark/q8.slt.part

Only test DATA is transcribed (the `from_pretty` literals, the executor configuration and the
push / expect script of each test); no reference code is copied.
"""
import json
import os
import re
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else ""
OUT = sys.argv[2] if len(sys.argv) > 2 else os.path.dirname(os.path.abspath(__file__))


def clean_pretty(lit: str) -> str:
    lines = [ln.strip() for ln in lit.split("\n")]
    return "\n".join(ln for ln in lines if ln)


def split_tests(src: str, start_marker: str = "#[tokio::test]"):
    parts = src.split(start_marker)[1:]
    for p in parts:
        m = re.search(r"async fn (\w+)\s*\(", p)
        if m:
            yield m.group(1), p


# ----------------------------------------------------------------------------------- hash join
def extract_hash_join():
    path = os.path.join(REF, "src/stream/src/executor/hash_join.rs")
    src = open(path).read()
    tests_start = src.index("#[cfg(test)]")
    src_tests = src[tests_start:]
    line_of = lambda pos: src[: tests_start + pos].count("\n") + 1  # noqa: E731
    out = []
    for name, body in split_tests(src_tests):
        pos0 = src_tests.index("async fn " + name)
        entry = {"name": name, "source": f"src/stream/src/executor/hash_join.rs:{line_of(pos0)}"}
        if "push_watermark" in body or "push_int64_watermark" in body or "InequalityPairInfo {" in body:
            entry["skipped"] = "watermark / inequality state cleaning stays on the CPU executor (SURVEY 8a)"
            out.append(entry)
            continue
        chunks = {m.group(1): clean_pretty(m.group(2))
                  for m in re.finditer(r"let (\w+) = StreamChunk::from_pretty\(\s*\"([^\"]*)\",?\s*(?://[^\n]*)?\s*\);", body)}
        mc = re.search(r"create_(classical_executor|append_only_executor|executor_with_evict_interval|executor)"
                       r"::<\{\s*JoinType::(\w+)\s*\}>\(([^;]*?)\)\s*\.await", body, re.S)
        assert mc, name
        kind, jt, args = mc.group(1), mc.group(2), mc.group(3)
        args = [a.strip() for a in args.split(",") if a.strip()]
        cfg = {"join_type": jt}
        if kind == "classical_executor":
            # create_classical_executor(with_condition, null_safe, condition_text) hash_join.rs:1628-1636
            cfg.update(schema="II", stream_key=[1], join_keys=[0], deduped_pk=[1], append_only=False,
                       null_safe=[args[1] == "true"],
                       cond="(less_than:boolean $1:int8 $3:int8)" if args[0] == "true" else None)
        elif kind == "append_only_executor":
            # create_append_only_executor(with_condition) hash_join.rs:1638-1718
            cfg.update(schema="III", stream_key=[0], join_keys=[0, 1], deduped_pk=[], append_only=True,
                       null_safe=[False, False],
                       cond="(less_than:boolean $1:int8 $3:int8)" if args[0] == "true" else None)
        elif kind == "executor_with_evict_interval":
            cfg.update(schema="II", stream_key=[1], join_keys=[0], deduped_pk=[1], append_only=False,
                       null_safe=[False], cond=None, evict_interval=int(args[0]))
        else:
            raise AssertionError((name, kind))
        entry["config"] = cfg
        # `let (mut tx_a, mut tx_b, mut hash_join) = create_..`: the FIRST sender is the left input
        # (test_streaming_hash_right_anti_join binds them swapped on purpose)
        mb = re.search(r"let \(mut tx_([lr]), mut tx_([lr]), mut hash_join\)", body)
        side_of = {mb.group(1): "l", mb.group(2): "r"}
        # the push / expect script, in source order
        pat = re.compile(
            r"tx_(?P<cs>[lr])\.push_chunk\((?:(?P<cv>\w+)\)|StreamChunk::from_pretty\(\s*\"(?P<cl>[^\"]*)\",?\s*\)\))"
            r"|tx_(?P<bs>[lr])\.push_barrier\(test_epoch\((?P<be>\d+)\),\s*(?:false|true)\)"
            r"|hash_join\.(?P<pend>next_unwrap_pending)\(\)"
            r"|hash_join\.(?P<rb>next_unwrap_ready_barrier)\(\)"
            r"|hash_join\.next_unwrap_ready_chunk\(\)\?;\s*(?P<cp>let chunk = chunk\.compact_vis\(\);)?\s*assert_eq!\(\s*chunk,\s*"
            r"StreamChunk::from_pretty\(\s*\"(?P<exp>[^\"]*)\"", re.S)
        steps = []
        for m in pat.finditer(body):
            if m.group("cs"):
                lit = chunks[m.group("cv")] if m.group("cv") else clean_pretty(m.group("cl"))
                steps.append({"op": "push_chunk", "side": side_of[m.group("cs")], "chunk": lit})
            elif m.group("bs"):
                steps.append({"op": "push_barrier", "side": side_of[m.group("bs")], "epoch": int(m.group("be"))})
            elif m.group("pend"):
                steps.append({"op": "expect_pending"})
            elif m.group("rb"):
                steps.append({"op": "expect_barrier"})
            else:
                st = {"op": "expect_chunk", "chunk": clean_pretty(m.group("exp"))}
                if m.group("cp"):
                    st["compact_vis"] = True
                steps.append(st)
        n_expect_src = body.count("next_unwrap_ready_chunk")
        n_expect = sum(1 for s in steps if s["op"] == "expect_chunk")
        assert n_expect == n_expect_src, (name, n_expect, n_expect_src)
        entry["steps"] = steps
        out.append(entry)
    return out


# ----------------------------------------------------------------------------------- hash agg
def parse_snapshot_table(block: str):
    rows = []
    for ln in block.split("\n"):
        ln = ln.strip()
        if ln.startswith("|"):
            cells = [c.strip() for c in ln.strip("|").split("|")]
            rows.append(cells)
    return rows


def extract_hash_agg():
    path = os.path.join(REF, "src/stream/tests/integration_tests/hash_agg.rs")
    src = open(path).read()
    out = []
    for name, body in split_tests(src):
        pos0 = src.index("async fn " + name)
        entry = {"name": name, "source": f"src/stream/tests/integration_tests/hash_agg.rs:{src[:pos0].count(chr(10)) + 1}"}
        if "emit_on_window_close" in body or "eowc" in name:
            entry["skipped"] = "EOWC sort buffer is out of GPU scope (hash_agg.rs:434-474)"
            out.append(entry)
            continue
        calls = re.findall(r"AggCall::from_pretty\(\"([^\"]*)\"\)", body)
        m = re.search(r"new_boxed_hash_agg_executor\(\s*store,\s*source,\s*(true|false)", body)
        append_only = m.group(1) == "true"
        n_fields = len(re.findall(r"Field::unnamed\(DataType::Int64\)", body))
        mk = re.search(r"let (?:key_indices|keys) = vec!\[([^\]]*)\]", body)
        keys = [int(x) for x in mk.group(1).split(",") if x.strip()]
        steps = []
        pat = re.compile(r"tx\.push_barrier\(test_epoch\((\d+)\),\s*false\)"
                         r"|tx\.push_chunk\(StreamChunk::from_pretty\(\s*\"([^\"]*)\",?\s*\)\)", re.S)
        for mm in pat.finditer(body):
            if mm.group(1):
                steps.append({"op": "push_barrier", "epoch": int(mm.group(1))})
            else:
                steps.append({"op": "push_chunk", "chunk": clean_pretty(mm.group(2))})
        snap = re.search(r"expect!\[\[r#\"(.*?)\"#\]\]", body, re.S).group(1)
        expected = []
        for ev in re.split(r"\n\s*- !", "\n" + snap)[1:]:
            if ev.startswith("barrier"):
                expected.append({"barrier": int(ev.split()[1])})
            elif ev.startswith("chunk"):
                rows = parse_snapshot_table(ev)
                expected.append({"chunk_rows": rows})
        entry.update(config={"schema": "I" * n_fields, "group_keys": keys, "agg_calls": calls,
                             "append_only": append_only, "row_count_index": 0},
                     steps=steps, expected=expected, sorted=True)
        if "min:int8" in "".join(calls) and not append_only:
            entry["retractable_min"] = True  # MaterializedInput state (minput.rs); offloaded since round 2
        out.append(entry)
    return out


# ----------------------------------------------------------------------------------- agg functions
def extract_agg_funcs():
    path = os.path.join(REF, "src/expr/impl/src/aggregate/general.rs")
    src = open(path).read()
    out = []
    # each #[test] fn holds one or more (input literal, test_agg(call, input, expected)) pairs
    for m in re.finditer(r"#\[test\]\s*fn (\w+)\(\)\s*\{(.*?)\n    \}", src, re.S):
        name, body = m.group(1), m.group(2)
        line = src[:m.start()].count(chr(10)) + 1
        pat = re.compile(r"StreamChunk::from_pretty\(\s*\"(?P<lit>[^\"]*)\",?\s*\)"
                         r"|test_agg\(\s*\"(?P<call>[^\"]*)\"\s*,\s*input\s*,\s*(?P<exp>.*?)\s*,?\s*\);", re.S)
        last = None
        k = 0
        for mm in pat.finditer(body):
            if mm.group("lit") is not None:
                last = clean_pretty(mm.group("lit"))
            else:
                out.append({"name": f"{name}#{k}", "source": f"src/expr/impl/src/aggregate/general.rs:{line}",
                            "call": mm.group("call"), "input": last,
                            "expected_expr": " ".join(mm.group("exp").split())})
                k += 1
    return out


# ----------------------------------------------------------------------------------- filter
def extract_filter():
    """src/stream/src/executor/filter.rs tests: input chunks, the predicate, expected output chunks"""
    path = os.path.join(REF, "src/stream/src/executor/filter.rs")
    src = open(path).read()
    tests_start = src.index("#[cfg(test)]")
    src_tests = src[tests_start:]
    line_of = lambda pos: src[: tests_start + pos].count("\n") + 1  # noqa: E731
    out = []
    for name, body in split_tests(src_tests):
        pos0 = src_tests.index("async fn " + name)
        lits = [clean_pretty(re.sub(r"//[^\n]*", "", m.group(1)))
                for m in re.finditer(r"StreamChunk::from_pretty\(\s*\"([^\"]*)\",?\s*\)", body)]
        mexpr = re.search(r"build_from_pretty\(\"([^\"]+)\"\)", body)
        n_in = len(re.findall(r"let chunk\d* = StreamChunk::from_pretty", body))
        assert mexpr and n_in >= 1 and len(lits) == 2 * n_in, name
        out.append({"name": name, "source": f"src/stream/src/executor/filter.rs:{line_of(pos0)}",
                    "upsert": "UpsertFilterExecutor::new" in body, "expr": mexpr.group(1),
                    "inputs": lits[:n_in], "expected": lits[n_in:]})
    return out


# ----------------------------------------------------------------------------------- project
def extract_project():
    """src/stream/src/executor/project/project_scalar.rs test_projection: input chunks, the expression, expected chunks;
    src/expr/impl/src/scalar/tumble.rs has no value tests, so tumble_* is pinned by restating :91-112 only."""
    path = os.path.join(REF, "src/stream/src/executor/project/project_scalar.rs")
    src = open(path).read()
    tests_start = src.index("#[cfg(test)]")
    src_tests = src[tests_start:]
    line_of = lambda pos: src[: tests_start + pos].count("\n") + 1  # noqa: E731
    out = []
    for name, body in split_tests(src_tests):
        if name != "test_projection":
            continue  # the watermark tests are about watermark derivation (host side)
        pos0 = src_tests.index("async fn " + name)
        lits = [clean_pretty(re.sub(r"//[^\n]*", "", m.group(1)))
                for m in re.finditer(r"StreamChunk::from_pretty\(\s*\"([^\"]*)\",?\s*\)", body)]
        exprs = re.findall(r"build_from_pretty\(\"([^\"]+)\"\)", body)
        n_in = len(re.findall(r"let chunk\d* = StreamChunk::from_pretty", body))
        assert exprs and n_in >= 1 and len(lits) == 2 * n_in, name
        out.append({"name": name, "source": f"src/stream/src/executor/project/project_scalar.rs:{line_of(pos0)}",
                    "exprs": exprs, "inputs": lits[:n_in], "expected": lits[n_in:]})
    return out


# ----------------------------------------------------------------------------------- nexmark e2e fixture (q4)
def extract_nexmark_q4():
    """e2e_test/nexmark/insert_{auction,bid}.slt.part + the expected rows of e2e_test/streaming/nexmark/q4.slt.part
    (view: e2e_test/streaming/nexmark/views/q4.slt.part).  Only the columns q4 reads are kept; timestamps become
    microseconds since the epoch (the in-memory representation of TIMESTAMP)."""
    import ast
    from datetime import datetime, timezone

    def ts(x):
        fmt = "%Y-%m-%d %H:%M:%S.%f" if "." in x else "%Y-%m-%d %H:%M:%S"
        d = datetime.strptime(x, fmt).replace(tzinfo=timezone.utc)
        return int(d.timestamp()) * 1_000_000 + d.microsecond

    def rows(path):
        out = []
        for ln in open(os.path.join(REF, path)):
            ln = ln.strip()
            if ln.startswith("(") and not ln.startswith("(\n") and ln[1:2].isdigit():
                out.append(ast.literal_eval(ln.rstrip(",;")))
        return out

    auction = [[r[0], ts(r[5]), ts(r[6]), r[8]] for r in rows("e2e_test/nexmark/insert_auction.slt.part")]   # id, date_time, expires, category
    bid = [[r[0], r[2], ts(r[5])] for r in rows("e2e_test/nexmark/insert_bid.slt.part")]                      # auction, price, date_time
    exp = []
    seen = False
    for ln in open(os.path.join(REF, "e2e_test/streaming/nexmark/q4.slt.part")):
        if ln.startswith("----"):
            seen = True
        elif seen and ln.strip():
            exp.append(ln.split())
    exp7, seen = [], False
    for ln in open(os.path.join(REF, "e2e_test/streaming/nexmark/q7.slt.part")):
        if ln.startswith("----"):
            seen = True
        elif seen and ln.strip():
            f = ln.split()
            exp7.append([int(f[0]), int(f[1]), int(f[2]), ts(f[3] + " " + f[4])])
    q7 = {"source": "e2e_test/nexmark/insert_bid.slt.part; view e2e_test/streaming/nexmark/views/q7.slt.part; expected "
                    "e2e_test/streaming/nexmark/q7.slt.part",
          "bid_columns": ["auction", "bidder", "price", "date_time_us"],
          "bid": [[r[0], r[1], r[2], ts(r[5])] for r in rows("e2e_test/nexmark/insert_bid.slt.part")],
          "expected_columns": ["auction", "price", "bidder", "date_time_us"], "expected_q7": exp7}
    json.dump(q7, open(os.path.join(OUT, "nexmark_q7_fixture.json"), "w"), indent=0)
    exp8, seen = [], False
    for ln in open(os.path.join(REF, "e2e_test/streaming/nexmark/q8.slt.part")):
        if ln.startswith("----"):
            seen = True
        elif seen and ln.strip():
            f = ln.rstrip("\n").split("\t")
            exp8.append([int(f[0]), f[1], ts(f[2])])
    q8 = {"source": "e2e_test/nexmark/insert_person.slt.part, insert_auction.slt.part; view e2e_test/streaming/nexmark/views/"
                    "q8.slt.part; expected e2e_test/streaming/nexmark/q8.slt.part",
          "person_columns": ["id", "name", "date_time_us"],
          "person": [[r[0], r[1], ts(r[6])] for r in rows("e2e_test/nexmark/insert_person.slt.part")],
          "auction_columns": ["seller", "date_time_us"],
          "auction": [[r[7], ts(r[5])] for r in rows("e2e_test/nexmark/insert_auction.slt.part")],
          "expected_columns": ["id", "name", "starttime_us"], "expected_q8": exp8}
    json.dump(q8, open(os.path.join(OUT, "nexmark_q8_fixture.json"), "w"), indent=0)
    return {"source": "e2e_test/nexmark/insert_auction.slt.part, insert_bid.slt.part; expected e2e_test/streaming/nexmark/q4.slt.part",
            "auction_columns": ["id", "date_time_us", "expires_us", "category"], "auction": auction,
            "bid_columns": ["auction", "price", "date_time_us"], "bid": bid, "expected_q4": exp}


def main():
    if not os.path.isdir(REF):
        sys.exit("usage: extract_ref_kats.py <risingwave checkout> [output directory]")
    hj = extract_hash_join()
    json.dump(hj, open(os.path.join(OUT, "hash_join_kats.json"), "w"), indent=1)
    ha = extract_hash_agg()
    json.dump(ha, open(os.path.join(OUT, "hash_agg_kats.json"), "w"), indent=1)
    af = extract_agg_funcs()
    json.dump(af, open(os.path.join(OUT, "agg_func_kats.json"), "w"), indent=1)
    q4 = extract_nexmark_q4()
    json.dump(q4, open(os.path.join(OUT, "nexmark_q4_fixture.json"), "w"), indent=0)
    print(f"nexmark q4 fixture: {len(q4['auction'])} auctions, {len(q4['bid'])} bids, {len(q4['expected_q4'])} expected rows")
    fl = extract_filter()
    json.dump(fl, open(os.path.join(OUT, "filter_kats.json"), "w"), indent=1)
    print(f"filter: {len(fl)} tests")
    pj = extract_project()
    json.dump(pj, open(os.path.join(OUT, "project_kats.json"), "w"), indent=1)
    print(f"project: {len(pj)} tests")
    print(f"hash_join: {len(hj)} tests ({sum('skipped' in t for t in hj)} skipped); "
          f"hash_agg: {len(ha)}; agg funcs: {len(af)}")


if __name__ == "__main__":
    main()
