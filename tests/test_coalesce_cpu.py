"""The request queue behind pb_search (next-plaid_b200/csrc/coalesce.h), on the host alone: a small harness drives it
from many threads with a fake batch function that records the groups it is given and can sleep or fail.  Every scenario
runs twice, built plainly and with -fsanitize=thread."""
import json
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "next-plaid_b200", "csrc")

HARNESS = r"""
#include "coalesce.h"
#include <cstdio>
#include <cstdlib>
#include <thread>

struct Req : pbq::Request {
    int payload = 0, result = -1;
    bool bad = false;  // refused when it runs alone, and refuses any batch it is in (as pb_search_batch_params does)
};
struct State {
    std::mutex m;
    std::vector<std::vector<int>> groups;
    int running = 0, max_running = 0, sleep_us = 0, fail_merged = 0;
    bool order_ok = true;
};
struct Fake {
    State *s;
    int operator()(pbq::Request *const *reqs, size_t n, std::string &err) const {
        bool any_bad = false;
        {
            std::lock_guard<std::mutex> g(s->m);
            std::vector<int> grp;
            for (size_t i = 0; i < n; ++i) {
                grp.push_back(static_cast<Req *>(reqs[i])->payload);
                any_bad = any_bad || static_cast<Req *>(reqs[i])->bad;
                if (i && reqs[i]->enqueued < reqs[i - 1]->enqueued) s->order_ok = false;
            }
            s->groups.push_back(grp);
            s->max_running = std::max(s->max_running, ++s->running);
        }
        if (s->sleep_us) std::this_thread::sleep_for(std::chrono::microseconds(s->sleep_us));
        {
            std::lock_guard<std::mutex> g(s->m);
            --s->running;
        }
        if (n > 1 && s->fail_merged) {
            err = "merged call failed";
            return s->fail_merged;
        }
        if (any_bad) {
            err = "bad request " + std::to_string(static_cast<Req *>(reqs[0])->payload);
            if (n > 1) err = "a bad request in the batch";
            return 7;
        }
        for (size_t i = 0; i < n; ++i) static_cast<Req *>(reqs[i])->result = 3 * static_cast<Req *>(reqs[i])->payload + 1;
        return 0;
    }
};

int main(int argc, char **argv) {
    if (argc != 11) return 2;
    const int T = atoi(argv[1]), R = atoi(argv[2]);
    pbq::Config cfg;
    cfg.max_queries = atoi(argv[3]), cfg.max_wait_us = atoi(argv[4]), cfg.max_inflight = atoi(argv[5]);
    State st;
    st.sleep_us = atoi(argv[6]), st.fail_merged = atoi(argv[7]);
    const int bad_every = atoi(argv[8]), refuse_every = atoi(argv[9]), fatal = atoi(argv[10]);
    pbq::Queue<Fake> q(Fake{&st}, fatal);
    q.configure(cfg);
    std::vector<int> status(T * R, -1), result(T * R, -1);
    std::vector<std::string> error(T * R);
    std::atomic<int> ready{0};
    std::vector<std::thread> th;
    for (int t = 0; t < T; ++t)
        th.emplace_back([&, t] {
            ++ready;
            while (ready.load() < T) std::this_thread::yield();
            for (int i = 0; i < R; ++i) {
                const int p = t * R + i + 1;
                if (refuse_every && p % refuse_every == 0) {  // the caller's own validation: never queued
                    q.count_refused();
                    status[p - 1] = 1;
                    continue;
                }
                Req r;
                r.payload = p;
                r.bad = bad_every && p % bad_every == 0;
                q.submit(r);
                status[p - 1] = r.status, result[p - 1] = r.result, error[p - 1] = r.error;
            }
        });
    for (auto &x : th) x.join();
    const pbq::Counters c = q.counters(false);
    printf("{\"groups\": [");
    for (size_t g = 0; g < st.groups.size(); ++g) {
        printf("%s[", g ? ", " : "");
        for (size_t i = 0; i < st.groups[g].size(); ++i) printf("%s%d", i ? ", " : "", st.groups[g][i]);
        printf("]");
    }
    printf("], \"status\": [");
    for (int i = 0; i < T * R; ++i) printf("%s%d", i ? ", " : "", status[i]);
    printf("], \"result\": [");
    for (int i = 0; i < T * R; ++i) printf("%s%d", i ? ", " : "", result[i]);
    printf("], \"error\": [");
    for (int i = 0; i < T * R; ++i) printf("%s\"%s\"", i ? ", " : "", error[i].c_str());
    printf("], \"max_running\": %d, \"order_ok\": %s, ", st.max_running, st.order_ok ? "true" : "false");
    printf("\"n_requests\": %lld, \"n_batches\": %lld, \"n_refused\": %lld, \"n_rerun_alone\": %lld, \"max_batch\": %lld, "
           "\"queue_wait_us\": %lld, \"batch_hist\": [",
           (long long)c.n_requests, (long long)c.n_batches, (long long)c.n_refused, (long long)c.n_rerun_alone,
           (long long)c.max_batch, (long long)c.queue_wait_us);
    for (int i = 0; i < 8; ++i) printf("%s%lld", i ? ", " : "", (long long)c.batch_hist[i]);
    printf("]}\n");
    return 0;
}
"""


@pytest.fixture(scope="module", params=["plain", "tsan"])
def harness(request, tmp_path_factory):
    cxx = shutil.which("g++")
    if not cxx:
        pytest.skip("no g++")
    d = tmp_path_factory.mktemp("coalesce_" + request.param)
    src, exe = d / "harness.cpp", d / "harness"
    src.write_text(HARNESS)
    flags = ["-std=c++17", "-O1", "-g", "-pthread", "-I", CSRC]
    if request.param == "tsan":
        flags += ["-fsanitize=thread"]
    r = subprocess.run([cxx] + flags + [str(src), "-o", str(exe)], capture_output=True, text=True)
    if r.returncode != 0:
        if request.param == "tsan":
            pytest.skip("the ThreadSanitizer runtime is not installed: " + r.stderr[-300:])
        raise AssertionError(r.stderr)
    env = dict(os.environ, TSAN_OPTIONS="exitcode=66 halt_on_error=0")

    def run(T, R, max_queries, max_wait_us=0, max_inflight=2, sleep_us=0, fail_merged=0, bad_every=0,
            refuse_every=0, fatal=2):
        args = [T, R, max_queries, max_wait_us, max_inflight, sleep_us, fail_merged, bad_every, refuse_every, fatal]
        p = subprocess.run([str(exe)] + [str(a) for a in args], capture_output=True, text=True, env=env, timeout=300)
        assert "ThreadSanitizer" not in p.stderr and p.returncode == 0, (p.returncode, p.stderr[-3000:])
        return json.loads(p.stdout)

    if request.param == "tsan":  # the runtime can be present and still unusable (address-space layout)
        p = subprocess.run([str(exe)] + ["1", "1", "1", "0", "1", "0", "0", "0", "0", "2"], capture_output=True,
                           text=True, env=env)
        if p.returncode != 0 and "data race" not in p.stderr:
            pytest.skip("the ThreadSanitizer runtime does not start here: " + p.stderr[-300:])
    return run


def served_once(out, n, skipped=()):
    seen = sorted(p for g in out["groups"] for p in g)
    return seen == [p for p in range(1, n + 1) if p not in skipped]


def hist_bucket(n):
    b = 0
    while b < 7 and (1 << b) < n:
        b += 1
    return b


def test_every_request_served_once_with_its_own_result(harness):
    T, R = 16, 40
    out = harness(T, R, max_queries=8, max_inflight=2, sleep_us=200)
    assert served_once(out, T * R)
    assert out["status"] == [0] * (T * R)
    assert out["result"] == [3 * p + 1 for p in range(1, T * R + 1)]
    assert max(len(g) for g in out["groups"]) <= 8 and out["max_batch"] <= 8
    assert out["max_running"] <= 2
    assert out["n_requests"] == T * R and out["n_batches"] == len(out["groups"]) and out["n_rerun_alone"] == 0
    hist = [0] * 8
    for g in out["groups"]:
        hist[hist_bucket(len(g))] += 1
    assert out["batch_hist"] == hist


def test_one_thread_never_waits_and_never_batches(harness):
    out = harness(1, 50, max_queries=32, max_wait_us=0, max_inflight=2)
    assert [len(g) for g in out["groups"]] == [1] * 50
    assert [g[0] for g in out["groups"]] == list(range(1, 51))
    assert out["max_running"] == 1 and out["batch_hist"][0] == 50


def test_one_inflight_batch_at_a_time(harness):
    out = harness(8, 30, max_queries=4, max_inflight=1, sleep_us=100)
    assert served_once(out, 240) and out["max_running"] == 1
    assert max(len(g) for g in out["groups"]) <= 4


def test_batches_form_behind_a_slow_batch_in_arrival_order(harness):
    # 32 threads behind batches of 2 ms each: while max_inflight batches run, the others can only queue
    out = harness(32, 6, max_queries=32, max_inflight=1, sleep_us=2000)
    assert served_once(out, 192)
    assert out["max_batch"] > 1 and any(len(g) > 1 for g in out["groups"])
    assert out["order_ok"]
    assert out["queue_wait_us"] > 0


def test_a_waiting_leader_gathers_company(harness):
    # nothing is slow here: batches can only form because the leader waits for the threads released together
    out = harness(8, 1, max_queries=8, max_wait_us=10000, max_inflight=2)
    assert served_once(out, 8)
    assert out["n_batches"] <= 8 and out["max_batch"] <= 8 and out["order_ok"]


def test_failed_merged_batch_reruns_members_alone(harness):
    # every merged call fails with a status that is not the fatal one; each member then runs alone and succeeds
    T, R = 16, 10
    out = harness(T, R, max_queries=8, max_inflight=2, sleep_us=300, fail_merged=5, fatal=2)
    assert out["status"] == [0] * (T * R)
    assert out["result"] == [3 * p + 1 for p in range(1, T * R + 1)]
    merged = [g for g in out["groups"] if len(g) > 1]
    assert merged and out["n_rerun_alone"] == sum(len(g) for g in merged)
    singles = sorted(g[0] for g in out["groups"] if len(g) == 1)
    assert singles == list(range(1, T * R + 1))      # alone exactly once, whether it was merged first or not


def test_bad_member_gets_its_own_status_and_neighbours_succeed(harness):
    T, R = 16, 10
    out = harness(T, R, max_queries=8, max_inflight=1, sleep_us=300, bad_every=7)
    for p in range(1, T * R + 1):
        if p % 7 == 0:
            assert out["status"][p - 1] == 7 and out["error"][p - 1] == f"bad request {p}" and out["result"][p - 1] == -1
        else:
            assert out["status"][p - 1] == 0 and out["result"][p - 1] == 3 * p + 1 and out["error"][p - 1] == ""


def test_device_failure_goes_to_every_member(harness):
    T, R = 16, 4
    out = harness(T, R, max_queries=16, max_inflight=1, sleep_us=2000, fail_merged=2, fatal=2)
    assert out["n_rerun_alone"] == 0
    failed = {p for g in out["groups"] if len(g) > 1 for p in g}
    assert failed
    for p in range(1, T * R + 1):
        if p in failed:
            assert out["status"][p - 1] == 2 and out["error"][p - 1] == "merged call failed"
        else:
            assert out["status"][p - 1] == 0 and out["result"][p - 1] == 3 * p + 1
    assert served_once(out, T * R)                    # nobody ran twice


def test_refused_request_never_reaches_the_batch_function(harness):
    T, R = 8, 20
    out = harness(T, R, max_queries=8, sleep_us=100, refuse_every=5)
    refused = [p for p in range(1, T * R + 1) if p % 5 == 0]
    assert served_once(out, T * R, skipped=set(refused))
    assert out["n_refused"] == len(refused) and out["n_requests"] == T * R - len(refused)
    assert all(out["status"][p - 1] == 1 for p in refused)
