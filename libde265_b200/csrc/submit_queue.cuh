// submit_queue.cuh — the queue behind b200_engine_submit_picture_async.
//
// b200_engine_submit_picture spends ~1 ms of host time per 4K picture (validation, work lists, packing), spread over the pool
// threads but with serial joins; a host that produces pictures faster than that (a parser with several slice / WPP threads, a
// cache of recorded pictures, bench.py's e2e leg) is held up by it.  The queue plans WHOLE pictures in parallel: N planner
// threads run the engine's `plan` step on one picture each; ONE sequencer thread takes the commands in submission order, waits
// for a picture's plan and runs the engine's `issue` step.  Read-backs are queued behind the pictures they follow.  Host code
// only, so tests/submit_queue_emul.cu tests it on the CPU; uses set_err / g_err / prof_now of the including translation unit.
#pragma once
#include <algorithm>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <exception>
#include <functional>
#include <mutex>
#include <sched.h>
#include <string>
#include <thread>
#include <vector>

#include "b200hevc.h"

#define B200_ASYNC_DEPTH 32  // queued pictures at most

enum class CmdKind { picture, read };
enum class CmdState { queued, planning, planned };

// One queued command.  The engine derives its payload (the picture, its layout and staging set, the read's planes) from it.
struct SubmitCmd {
  CmdKind kind = CmdKind::picture;
  int slot = -1;                     // the slot the picture writes or the read-back reads
  CmdState state = CmdState::queued;  // guarded by SubmitQueue::m
  unsigned long long ticket = 0;     // position in submission order (1, 2, ...)
  int rc = B200_OK;
  std::string err;                   // the failing thread's g_err
  double plan_s = 0;                 // B200_HOST_PROF: planner thread time
  virtual ~SubmitCmd() = default;
};

// Cores this process may use: the affinity mask, clamped by the cgroup v2 CPU quota.
static int host_cores()
{
  int n = (int)std::thread::hardware_concurrency();
  cpu_set_t set;
  if (sched_getaffinity(0, sizeof(set), &set) == 0) n = CPU_COUNT(&set);
  if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
    char quota[32] = "";
    long period = 0;
    if (fscanf(f, "%31s %ld", quota, &period) == 2 && strcmp(quota, "max") != 0 && period > 0) n = std::min(n, std::max(1, (int)((atol(quota) + period - 1) / period)));
    fclose(f);
  }
  return std::max(1, n);
}

struct SubmitQueue {
  // The engine's steps: plan a picture on planner thread `planner` (0 .. n-1), issue a command on the sequencer in ticket order,
  // and what each thread the queue starts runs first.
  std::function<int(int planner, SubmitCmd&)> plan;
  std::function<int(SubmitCmd&)> issue;
  std::function<void()> thread_start;
  static constexpr unsigned long long all = ~0ull;  // wait(all): everything queued so far

  // B200_HOST_PROF (set before start): the sequencer's view of the pictures once the warm-up counter *prof_skip (first-use
  // allocations; the engine's synchronous path counts down the same one) has run out.  Only the sequencer writes them.
  bool prof_on = false;
  int* prof_skip = nullptr;
  struct Prof {
    double plan_busy = 0, wait_plan = 0, issue_pictures = 0, issue_reads = 0;  // plan_busy: planner threads, summed
    unsigned long long pictures = 0;
  } prof;

  ~SubmitQueue() { stop(); }

  // One planner takes ~4 ms of one core per 4K picture: the cores this process may use (affinity mask and cgroup quota:
  // exceeding the quota gets the whole process throttled) minus four for the caller, the sequencer and the CUDA driver's threads,
  // at most 16 (B200_ASYNC_THREADS overrides).
  static int planner_threads()
  {
    int n = std::max(2, std::min(16, host_cores() - 4));
    if (const char* e = getenv("B200_ASYNC_THREADS")) n = std::max(1, std::min(32, atoi(e)));
    return n;
  }

  // Starts the sequencer and `n` planner threads (plan() sees planner indices 0 .. n-1).
  int start(int n)
  {
    depth = std::min(B200_ASYNC_DEPTH, n + 8);
    if (const char* e = getenv("B200_ASYNC_QUEUE")) depth = std::max(1, std::min(B200_ASYNC_DEPTH, atoi(e)));
    try {  // thread creation may throw (resource limits): no exception leaves the C ABI
      sequencer = std::thread([this] { run_sequencer(); });
      for (int w = 0; w < n; w++) planners.emplace_back([this, w] { run_planner(w); });
    } catch (const std::exception& ex) {
      if (planners.empty() || !sequencer.joinable()) {  // nothing usable: tear down what exists
        stop();
        return set_err(B200_ERR_NOMEM, "asynchronous submission: cannot start threads (%s)", ex.what());
      }
      // fewer planners than asked for still work
      depth = std::min(depth, (int)planners.size() + 8);
    }
    return B200_OK;
  }

  // Queues `cmd` (the queue deletes it once issued) behind `depth` pictures / 4 * B200_ASYNC_DEPTH commands at most; returns its ticket.
  unsigned long long enqueue(SubmitCmd* cmd)
  {
    {
      std::unique_lock<std::mutex> lk(m);
      cv_done.wait(lk, [&] { return n_pictures < depth && q.size() < 4 * B200_ASYNC_DEPTH; });
      cmd->ticket = ++enq_seq;
      q.push_back(cmd);
      if (cmd->kind == CmdKind::picture) n_pictures++;
      if (cmd->slot >= 0 && cmd->slot < B200_MAX_SLOTS) slot_seq[cmd->slot] = cmd->ticket;
    }
    if (cmd->kind == CmdKind::picture) cv_plan.notify_one();
    cv_seq.notify_all();
    return cmd->ticket;
  }

  unsigned long long last_ticket()
  {
    std::lock_guard<std::mutex> lk(m);
    return enq_seq;
  }

  // The ticket of the last queued command that writes or reads `slot` (0: none).
  unsigned long long slot_ticket(int slot)
  {
    std::lock_guard<std::mutex> lk(m);
    return slot_seq[slot];
  }

  // Blocks until every command up to `ticket` has been issued (a ticket never handed out: everything queued so far); returns
  // (and clears) the first error of a queued command — which may be that of a command after `ticket` retired meanwhile.
  int wait(unsigned long long ticket)
  {
    std::unique_lock<std::mutex> lk(m);
    ticket = std::min(ticket, enq_seq);
    cv_done.wait(lk, [&] { return done_seq >= ticket; });
    const int rc = first_rc;
    if (rc) set_err(rc, "%s", first_err.c_str());
    first_rc = B200_OK;
    first_err.clear();
    return rc;
  }

  // Issues what is queued, then joins every thread.
  void stop()
  {
    wait(all);
    {
      std::lock_guard<std::mutex> lk(m);
      stopping = true;
    }
    cv_plan.notify_all();
    cv_seq.notify_all();
    for (auto& t : planners) t.join();
    planners.clear();
    if (sequencer.joinable()) sequencer.join();
  }

  // Whether the picture being issued is profiled (B200_HOST_PROF, past the warm-up); read on the sequencer thread.
  bool profiling() const { return prof_on && *prof_skip <= 0; }

 private:
  std::mutex m;
  std::condition_variable cv_plan, cv_seq, cv_done;
  std::deque<SubmitCmd*> q;  // submission order; the front is the next one the sequencer issues
  int n_pictures = 0;        // pictures in q (read-backs do not count towards the depth)
  int depth = 12;            // pictures queued at most (B200_ASYNC_QUEUE; <= B200_ASYNC_DEPTH)
  std::vector<std::thread> planners;
  std::thread sequencer;
  bool stopping = false;
  int first_rc = B200_OK;
  std::string first_err;
  unsigned long long enq_seq = 0, done_seq = 0;      // tickets: queued last / issued last
  unsigned long long slot_seq[B200_MAX_SLOTS] = {};  // ticket of the last queued command that writes or reads the slot

  void run_planner(int w)
  {
    thread_start();
    for (;;) {
      SubmitCmd* cmd = nullptr;
      {
        std::unique_lock<std::mutex> lk(m);
        cv_plan.wait(lk, [&] {
          for (SubmitCmd* c : q)
            if (c->kind == CmdKind::picture && c->state == CmdState::queued) { cmd = c; return true; }
          return stopping;
        });
        if (!cmd) return;  // stopping
        cmd->state = CmdState::planning;
      }
      const double t0 = prof_on ? prof_now() : 0.0;
      const int rc = plan(w, *cmd);
      const double t1 = prof_on ? prof_now() : 0.0;
      {
        std::lock_guard<std::mutex> lk(m);
        cmd->plan_s = t1 - t0;
        cmd->rc = rc;
        if (rc) cmd->err = g_err;
        cmd->state = CmdState::planned;
      }
      cv_seq.notify_all();
    }
  }

  void run_sequencer()
  {
    thread_start();
    for (;;) {
      SubmitCmd* cmd = nullptr;
      double t0 = 0;
      {
        std::unique_lock<std::mutex> lk(m);
        cv_seq.wait(lk, [&] { return stopping || !q.empty(); });  // an empty queue is idle time, not waiting for a plan
        if (stopping) return;
        if (prof_on) t0 = prof_now();
        cv_seq.wait(lk, [&] { return stopping || (!q.empty() && (q.front()->kind == CmdKind::read || q.front()->state == CmdState::planned)); });
        if (stopping) return;
        cmd = q.front();
      }
      const bool picture = cmd->kind == CmdKind::picture;
      const double t1 = prof_on ? prof_now() : 0.0;
      int rc = cmd->rc;
      if (!rc) {
        rc = issue(*cmd);
        if (rc) cmd->err = g_err;
      }
      if (prof_on && *prof_skip > 0) {
        if (picture) (*prof_skip)--;
      } else if (prof_on) {
        (picture ? prof.issue_pictures : prof.issue_reads) += prof_now() - t1;
        prof.wait_plan += t1 - t0;
        if (picture) {
          prof.plan_busy += cmd->plan_s;
          prof.pictures++;
        }
      }
      {
        std::lock_guard<std::mutex> lk(m);
        if (rc && !first_rc) { first_rc = rc; first_err = cmd->err; }
        q.pop_front();
        if (picture) n_pictures--;
        done_seq = cmd->ticket;
      }
      delete cmd;
      cv_done.notify_all();
    }
  }
};
