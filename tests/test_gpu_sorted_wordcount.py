"""SortedWordCount (WordCount with a first-letter key-range partitionfn) through the mirrored server:loop() on the
test.sh golden corpus: finalfn sees exactly the golden counts, in one ascending key order, and result partition k
holds exactly the words bisect_right over the splitters puts there."""
import bisect

import pytest

import mrhbm_loader
from conftest import expand_tokens

mrhbm_loader.load()
from lua_mapreduce_b200.mapreduce import server  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.SortedWordCount import init as SWC  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.WordCount import init as WordCount  # noqa: E402

S = "lua_mapreduce_b200.mapreduce.examples.SortedWordCount"


@pytest.mark.gpu
@pytest.mark.parametrize("combiner", [False, True])
def test_sorted_wordcount_on_gpu(tmp_path, golden_wordcount, combiner):
    files = []
    for job in range(4):
        toks = expand_tokens(golden_wordcount, job)
        p = tmp_path / ("file%d.txt" % job)
        p.write_bytes(b"\n".join(b" ".join(toks[i:i + 7]) for i in range(0, len(toks), 7)) + b"\n")
        files.append(str(p))
    WordCount.FILES[:] = files
    del SWC.RESULT[:]
    params = dict(taskfn=S + ".init", mapfn=S + ".init", partitionfn=S + ".partitionfn", reducefn=S + ".init",
                  finalfn=S + ".finalfn", storage="hbm")
    if combiner:
        params["combinerfn"] = S + ".init"
    s = server.new("hbm://local", "sorted-wc-%d" % combiner)
    s.configure(params)
    s.loop()
    want = sorted((k, sum(c)) for k, _, c in golden_wordcount)
    assert SWC.RESULT == want  # every word once, ascending across all partitions
    spl = [x.encode() for x in SWC.hbm_splitters]
    for j in s.results:
        p = int(j["_id"])
        for key, _ in j["value"]["pairs"]:
            assert bisect.bisect_right(spl, key) == p == SWC.partitionfn(key)
