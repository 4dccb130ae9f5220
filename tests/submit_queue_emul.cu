// submit_queue_emul.cu — TEST INFRASTRUCTURE: drives the asynchronous submission queue (libde265_b200/csrc/submit_queue.cuh,
// the very code behind b200_engine_submit_picture_async) with stand-in plan and issue steps, so that
// tests/test_cpu_submit_queue.py checks its contract without a GPU: issue order, tickets, per-slot tickets, queued errors,
// back-pressure and shutdown.  The plan step sleeps, can wait on a gate and can fail; the issue step logs (ticket, kind, slot)
// and can fail.  Built by the test with nvcc as a host-only shared library (tests/libsubmit_queue_emul.so); not part of the
// product.
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <sys/syscall.h>
#include <unistd.h>
#include <thread>
#include <vector>

static thread_local char g_err[512] = "";
static int set_err(int code, const char* fmt, ...)
{
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
static inline double prof_now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

#include "submit_queue.cuh"

#define EXPORT extern "C" __attribute__((visibility("default")))

enum { FAIL_PLAN = 1, FAIL_ISSUE = 2 };

struct EmulCmd : SubmitCmd {
  int plan_us = 0, flags = 0;
  int gate = 0;         // > 0: the plan waits until sq_open_gate(gate)
  int hold_until = 0;   // > 0: the plan waits until that many enqueue calls have returned and the caller is blocked in the next
};

struct Emul {
  SubmitQueue q;
  std::mutex m;
  std::condition_variable cv;
  bool gate_open[16] = {};
  bool closing = false;
  int gate_timeouts = 0;
  std::vector<unsigned long long> log_ticket, plan_done;
  std::vector<int> log_kind, log_slot;
  std::atomic<int> thread_starts{0}, live{0};  // live: threads of the queue that have started and not yet exited
  std::atomic<int> entered{0}, returned{0};    // enqueue calls begun / returned
  std::atomic<long> caller{0};                  // the thread that called enqueue last
  int issued = 0, max_queued = 0;  // sequencer only

  // Waits (at most 5 s, so that a broken queue fails instead of hanging) until `ready` holds.
  template <class F> void hold(F ready)
  {
    std::unique_lock<std::mutex> lk(m);
    if (!cv.wait_for(lk, std::chrono::seconds(5), [&] { return closing || ready(); })) gate_timeouts++;
  }

  // Until `n` enqueue calls have returned and the caller sleeps in the next one (the queue is full), or that one returned too (a
  // queue that takes more than it should).  Polls: a thread falling asleep sends no notify.
  void hold_until_caller_blocked(int n)
  {
    for (int i = 0; i < 5000; i++) {
      if (returned > n) return;
      // asleep between entering call n + 1 and returning from it: blocked in the queue's enqueue
      if (entered > n && sleeping(caller) && returned == n) return;
      {
        std::lock_guard<std::mutex> lk(m);
        if (closing) return;
      }
      std::this_thread::sleep_for(std::chrono::milliseconds(1));
    }
    std::lock_guard<std::mutex> lk(m);
    gate_timeouts++;
  }

  static bool sleeping(long tid)  // the thread's state in /proc: S = waiting (here: on the queue's lock or condition)
  {
    char path[64], buf[256] = "";
    snprintf(path, sizeof(path), "/proc/self/task/%ld/stat", tid);
    FILE* f = fopen(path, "r");
    if (!f) return false;
    const size_t n = fread(buf, 1, sizeof(buf) - 1, f);
    fclose(f);
    const char* p = strrchr(buf, ')');  // "tid (comm) state ..."
    return n && p && p[1] == ' ' && p[2] == 'S';
  }
};

// Counts a queue thread as live from its start step until it exits (thread-local destructors run before join returns).
struct LiveThread {
  Emul* e = nullptr;
  ~LiveThread() { if (e) e->live--; }
};
static thread_local LiveThread t_live;

EXPORT void* sq_create(int n_planners)
{
  Emul* e = new Emul();
  e->q.thread_start = [e] {
    e->thread_starts++;
    e->live++;
    t_live.e = e;
  };
  e->q.plan = [e](int w, SubmitCmd& c) -> int {
    EmulCmd& cmd = static_cast<EmulCmd&>(c);
    if (cmd.gate) e->hold([&] { return e->gate_open[cmd.gate]; });
    if (cmd.hold_until) e->hold_until_caller_blocked(cmd.hold_until);
    std::this_thread::sleep_for(std::chrono::microseconds(cmd.plan_us));
    {
      std::lock_guard<std::mutex> lk(e->m);
      e->plan_done.push_back(cmd.ticket);
    }
    if (cmd.flags & FAIL_PLAN) return set_err(B200_ERR_INVALID, "plan of ticket %llu failed on planner %d", cmd.ticket, w);
    return B200_OK;
  };
  e->q.issue = [e](SubmitCmd& c) -> int {
    // every command the queue holds was enqueued; the ones issued before this one have left it
    e->max_queued = std::max(e->max_queued, e->returned.load() - e->issued);
    e->issued++;
    if (static_cast<EmulCmd&>(c).flags & FAIL_ISSUE) return set_err(B200_ERR_CUDA, "issue of ticket %llu failed", c.ticket);
    std::lock_guard<std::mutex> lk(e->m);
    e->log_ticket.push_back(c.ticket);
    e->log_kind.push_back((int)c.kind);
    e->log_slot.push_back(c.slot);
    return B200_OK;
  };
  if (e->q.start(n_planners)) { delete e; return nullptr; }
  return e;
}

EXPORT void sq_destroy(void* h)
{
  Emul* e = (Emul*)h;
  {
    std::lock_guard<std::mutex> lk(e->m);
    e->closing = true;  // release every gate
  }
  e->cv.notify_all();
  e->q.stop();
  delete e;
}

static unsigned long long enqueue(Emul* e, EmulCmd* cmd)
{
  e->caller = syscall(SYS_gettid);
  e->entered++;
  const unsigned long long t = e->q.enqueue(cmd);
  e->returned++;
  return t;
}

EXPORT unsigned long long sq_picture(void* h, int slot, int plan_us, int flags, int gate, int hold_until)
{
  EmulCmd* cmd = new EmulCmd();
  cmd->slot = slot;
  cmd->plan_us = plan_us;
  cmd->flags = flags;
  cmd->gate = gate;
  cmd->hold_until = hold_until;
  return enqueue((Emul*)h, cmd);
}

EXPORT unsigned long long sq_read(void* h, int slot, int flags)
{
  EmulCmd* cmd = new EmulCmd();
  cmd->kind = CmdKind::read;
  cmd->slot = slot;
  cmd->flags = flags;
  return enqueue((Emul*)h, cmd);
}

EXPORT void sq_open_gate(void* h, int gate)
{
  Emul* e = (Emul*)h;
  {
    std::lock_guard<std::mutex> lk(e->m);
    e->gate_open[gate] = true;
  }
  e->cv.notify_all();
}

EXPORT int sq_wait(void* h, unsigned long long ticket) { return ((Emul*)h)->q.wait(ticket); }
EXPORT unsigned long long sq_last_ticket(void* h) { return ((Emul*)h)->q.last_ticket(); }
EXPORT unsigned long long sq_slot_ticket(void* h, int slot) { return ((Emul*)h)->q.slot_ticket(slot); }
EXPORT void sq_stop(void* h) { ((Emul*)h)->q.stop(); }
EXPORT const char* sq_last_error() { return g_err; }
EXPORT int sq_total_limit() { return 4 * B200_ASYNC_DEPTH; }
EXPORT int sq_thread_starts(void* h) { return ((Emul*)h)->thread_starts.load(); }
EXPORT int sq_live_threads(void* h) { return ((Emul*)h)->live.load(); }
EXPORT int sq_max_queued(void* h) { return ((Emul*)h)->max_queued; }  // after a wait: the sequencer is idle

EXPORT int sq_gate_timeouts(void* h)
{
  Emul* e = (Emul*)h;
  std::lock_guard<std::mutex> lk(e->m);
  return e->gate_timeouts;
}

// The issue log so far: n entries of (ticket, kind 0 picture / 1 read, slot); returns n.
EXPORT int sq_log(void* h, unsigned long long* tickets, int* kinds, int* slots, int cap)
{
  Emul* e = (Emul*)h;
  std::lock_guard<std::mutex> lk(e->m);
  const int n = (int)e->log_ticket.size();
  for (int i = 0; i < n && i < cap; i++) { tickets[i] = e->log_ticket[i]; kinds[i] = e->log_kind[i]; slots[i] = e->log_slot[i]; }
  return n;
}

// The tickets of the pictures in the order their plans finished; returns n.
EXPORT int sq_plan_order(void* h, unsigned long long* tickets, int cap)
{
  Emul* e = (Emul*)h;
  std::lock_guard<std::mutex> lk(e->m);
  const int n = (int)e->plan_done.size();
  for (int i = 0; i < n && i < cap; i++) tickets[i] = e->plan_done[i];
  return n;
}
