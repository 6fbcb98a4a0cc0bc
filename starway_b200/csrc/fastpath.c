/* starway_b200 — CPython fast path for the binding layer (NOT part of the compute path).
 *
 * The reference reaches its engine through nanobind (C++), so its per-operation cost in the
 * binding is ~1 us.  A pure-ctypes shim costs ~3.5 us per asend/arecv and ~1.5 us per completion,
 * which caps the API-level message rate.  This module does the same three things the Python shim
 * does — resolve the buffer, call sw_post_send / sw_post_recv, resolve asyncio futures from
 * sw_poll — in C under the GIL.  It holds no engine logic: the function pointers it calls are the
 * C-ABI entry points of whichever library `_core.bind()` was given.  Without it `_core.py` falls
 * back to its ctypes implementation of the same steps.
 */
#define PY_SSIZE_T_CLEAN
#include <Python.h>
#include <stddef.h>
#include <structmember.h>
#include <stdint.h>
#include <string.h>

typedef struct {
  uint64_t op_id;
  int32_t status;
  uint32_t kind;
  uint64_t sender_tag;
  uint64_t length;
  uint64_t worker;
  uint64_t ep;
} sw_completion;

typedef uint64_t (*post_send_fn)(void*, uint64_t, uint64_t, const void*, size_t, uint64_t, int);
typedef uint64_t (*post_recv_fn)(void*, uint64_t, void*, size_t, uint64_t, uint64_t, int);
typedef int (*poll_fn)(void*, sw_completion*, int);

enum { SW_OP_RECV = 2 };

/* Pending fast-path operations: op id -> (loop, future, keep-alive), open addressing with linear
 * probing; keeping the entries in C saves a PyLong key, a 5-tuple and a dict insert + delete per
 * operation.  The engine hands out SEQUENTIAL op ids: hashed by `op & mask` thousands of
 * pre-posted receives would form one contiguous cluster and every deletion would scan all of it
 * (the cost of a completion grows with the number of receives outstanding), so the ids are scattered
 * with a multiplicative (Fibonacci) hash. */
typedef struct {
  uint64_t op; /* 0: empty */
  PyObject* loop;
  PyObject* fut;
  PyObject* keep;
} OpSlot;

typedef struct {
  PyObject_HEAD
  OpSlot* tab;
  size_t tab_cap; /* power of two */
  size_t tab_count;
  unsigned tab_shift; /* 64 - log2(tab_cap) */
  post_send_fn post_send;
  post_recv_fn post_recv;
  poll_fn poll;
  void* ctx;
  PyObject* ops;            /* dict shared with the Python shim: op id -> ("fut", loop, fut, keep, post_ok) */
  PyObject* resolve;        /* resolve(obj, writable) -> (ptr, nbytes, mem, keep)    [slow path: as_buffer] */
  PyObject* ensure_reader;  /* ensure_reader(loop) */
  PyObject* slow;           /* slow(entry, kind, status, sender_tag, length, worker, ep, here_loop, op_id) */
  PyObject* last_error;     /* last_error() -> str */
  PyObject* status_string;  /* status_string(code) -> str */
  PyObject* get_running_loop;
  PyObject* cache;          /* id(obj) -> (weakref, ptr, nbytes, mem, writable) */
  PyObject* last_loop;      /* loop whose reader registration was already ensured (borrowed identity) */
  PyObject* str_fut;        /* interned "fut" */
  PyObject* str_create_future;
  PyObject* str_set_result;
  PyObject* str_set_exception;
  PyObject* kick;           /* kick(): start polling the completion queue from the running loop (None until set) */
  int spinning;             /* set by the Python shim while the loop polls: a post then needs no kick */
  int closed;               /* set by the Python shim before the context goes away: Post objects then take the slow path */
} Binding;

static void tab_clear(Binding* self) {
  for (size_t i = 0; i < self->tab_cap; i++) {
    if (self->tab[i].op) {
      Py_XDECREF(self->tab[i].loop);
      Py_XDECREF(self->tab[i].fut);
      Py_XDECREF(self->tab[i].keep);
    }
  }
  PyMem_Free(self->tab);
  self->tab = NULL;
  self->kick = NULL;
  self->spinning = 0;
  self->closed = 0;
  self->tab_cap = self->tab_count = 0;
}

static inline size_t tab_home(uint64_t op, unsigned shift) { return (size_t)((op * 0x9E3779B97F4A7C15ull) >> shift); }

static OpSlot* tab_find(Binding* self, uint64_t op) {
  if (!self->tab_count || !op) return NULL; /* op 0: accept notifications carry no operation */
  const size_t mask = self->tab_cap - 1;
  for (size_t i = tab_home(op, self->tab_shift);; i = (i + 1) & mask) {
    if (self->tab[i].op == op) return &self->tab[i];
    if (self->tab[i].op == 0) return NULL;
  }
}

static void tab_place(OpSlot* tab, size_t mask, unsigned shift, OpSlot v) {
  size_t i = tab_home(v.op, shift);
  while (tab[i].op) i = (i + 1) & mask;
  tab[i] = v;
}

/* takes new references to loop / fut / keep */
static int tab_insert(Binding* self, uint64_t op, PyObject* loop, PyObject* fut, PyObject* keep) {
  if ((self->tab_count + 1) * 2 > self->tab_cap) {
    const size_t ncap = self->tab_cap ? self->tab_cap * 2 : 1024;
    unsigned nshift = 64;
    for (size_t c = ncap; c > 1; c >>= 1) nshift--;
    OpSlot* nt = (OpSlot*)PyMem_Calloc(ncap, sizeof(OpSlot));
    if (!nt) {
      PyErr_NoMemory();
      return -1;
    }
    for (size_t i = 0; i < self->tab_cap; i++)
      if (self->tab[i].op) tab_place(nt, ncap - 1, nshift, self->tab[i]);
    PyMem_Free(self->tab);
    self->tab = nt;
    self->tab_cap = ncap;
    self->tab_shift = nshift;
  }
  OpSlot v = {op, loop, fut, keep};
  Py_INCREF(loop);
  Py_INCREF(fut);
  Py_INCREF(keep);
  tab_place(self->tab, self->tab_cap - 1, self->tab_shift, v);
  self->tab_count++;
  return 0;
}

/* removes *s (its references now belong to the caller): backward-shift deletion */
static void tab_remove(Binding* self, OpSlot* s) {
  const size_t mask = self->tab_cap - 1;
  size_t i = (size_t)(s - self->tab), j = i;
  for (;;) {
    j = (j + 1) & mask;
    if (self->tab[j].op == 0) break;
    const size_t k = tab_home(self->tab[j].op, self->tab_shift); /* home position of the entry at j */
    const int stays = (i <= j) ? (i < k && k <= j) : (i < k || k <= j);
    if (stays) continue;
    self->tab[i] = self->tab[j];
    i = j;
  }
  self->tab[i].op = 0;
  self->tab_count--;
}

static void Binding_dealloc(Binding* self) {
  tab_clear(self);
  Py_XDECREF(self->ops);
  Py_XDECREF(self->resolve);
  Py_XDECREF(self->ensure_reader);
  Py_XDECREF(self->slow);
  Py_XDECREF(self->last_error);
  Py_XDECREF(self->status_string);
  Py_XDECREF(self->get_running_loop);
  Py_XDECREF(self->cache);
  Py_XDECREF(self->last_loop);
  Py_XDECREF(self->str_fut);
  Py_XDECREF(self->str_create_future);
  Py_XDECREF(self->str_set_result);
  Py_XDECREF(self->str_set_exception);
  Py_XDECREF(self->kick);
  Py_TYPE(self)->tp_free((PyObject*)self);
}

static int Binding_init(Binding* self, PyObject* args, PyObject* kw) {
  unsigned long long ps, pr, pl, ctx;
  PyObject *ops, *resolve, *ensure_reader, *slow, *last_error, *status_string;
  if (!PyArg_ParseTuple(args, "KKKKO!OOOOO", &ps, &pr, &pl, &ctx, &PyDict_Type, &ops, &resolve, &ensure_reader, &slow,
                        &last_error, &status_string))
    return -1;
  self->tab = NULL;
  self->kick = NULL;
  self->spinning = 0;
  self->closed = 0;
  self->tab_cap = self->tab_count = 0;
  self->tab_shift = 63;
  self->post_send = (post_send_fn)(uintptr_t)ps;
  self->post_recv = (post_recv_fn)(uintptr_t)pr;
  self->poll = (poll_fn)(uintptr_t)pl;
  self->ctx = (void*)(uintptr_t)ctx;
  Py_INCREF(ops);
  self->ops = ops;
  Py_INCREF(resolve);
  self->resolve = resolve;
  Py_INCREF(ensure_reader);
  self->ensure_reader = ensure_reader;
  Py_INCREF(slow);
  self->slow = slow;
  Py_INCREF(last_error);
  self->last_error = last_error;
  Py_INCREF(status_string);
  self->status_string = status_string;
  PyObject* asyncio = PyImport_ImportModule("asyncio");
  if (!asyncio) return -1;
  self->get_running_loop = PyObject_GetAttrString(asyncio, "get_running_loop");
  Py_DECREF(asyncio);
  if (!self->get_running_loop) return -1;
  self->cache = PyDict_New();
  self->last_loop = NULL;
  self->str_fut = PyUnicode_InternFromString("fut");
  self->str_create_future = PyUnicode_InternFromString("create_future");
  self->str_set_result = PyUnicode_InternFromString("set_result");
  self->str_set_exception = PyUnicode_InternFromString("set_exception");
  if (!self->cache || !self->str_fut || !self->str_create_future || !self->str_set_result || !self->str_set_exception)
    return -1;
  return 0;
}

/* -> 0 ok, -1 error.  keep is a NEW reference. */
static int resolve_buffer(Binding* self, PyObject* obj, int writable, void** ptr, size_t* nbytes, int* mem,
                          PyObject** keep) {
  PyObject* key = PyLong_FromVoidPtr(obj);
  if (!key) return -1;
  PyObject* hit = PyDict_GetItemWithError(self->cache, key); /* borrowed */
  if (hit) {
    PyObject* ref = PyTuple_GET_ITEM(hit, 0);
    PyObject* target = NULL;
#if PY_VERSION_HEX >= 0x030D0000
    if (PyWeakref_GetRef(ref, &target) < 0) target = NULL;
#else
    target = PyWeakref_GetObject(ref);
    Py_XINCREF(target);
#endif
    if (target == obj && (!writable || PyTuple_GET_ITEM(hit, 4) == Py_True)) {
      Py_DECREF(target);
      *ptr = PyLong_AsVoidPtr(PyTuple_GET_ITEM(hit, 1));
      *nbytes = PyLong_AsSize_t(PyTuple_GET_ITEM(hit, 2));
      *mem = (int)PyLong_AsLong(PyTuple_GET_ITEM(hit, 3));
      Py_DECREF(key);
      Py_INCREF(obj);
      *keep = obj;
      return 0;
    }
    Py_XDECREF(target);
  } else if (PyErr_Occurred()) {
    Py_DECREF(key);
    return -1;
  }
  /* slow path: the Python shim validates / converts (dtype, contiguity, device) */
  PyObject* res = PyObject_CallFunctionObjArgs(self->resolve, obj, writable ? Py_True : Py_False, NULL);
  if (!res) {
    Py_DECREF(key);
    return -1;
  }
  if (!PyTuple_Check(res) || PyTuple_GET_SIZE(res) != 4) {
    Py_DECREF(res);
    Py_DECREF(key);
    PyErr_SetString(PyExc_TypeError, "resolve() must return (ptr, nbytes, mem, keep)");
    return -1;
  }
  *ptr = PyLong_AsVoidPtr(PyTuple_GET_ITEM(res, 0));
  *nbytes = PyLong_AsSize_t(PyTuple_GET_ITEM(res, 1));
  *mem = (int)PyLong_AsLong(PyTuple_GET_ITEM(res, 2));
  *keep = PyTuple_GET_ITEM(res, 3);
  Py_INCREF(*keep);
  if (PyErr_Occurred()) {
    Py_DECREF(*keep);
    Py_DECREF(res);
    Py_DECREF(key);
    return -1;
  }
  /* cache only when the buffer object itself is what stays alive (no conversion happened) */
  if (*keep == obj) {
    PyObject* ref = PyWeakref_NewRef(obj, NULL);
    if (ref) {
      if (PyDict_GET_SIZE(self->cache) > 16384) PyDict_Clear(self->cache);
      PyObject* ent = PyTuple_Pack(5, ref, PyTuple_GET_ITEM(res, 0), PyTuple_GET_ITEM(res, 1), PyTuple_GET_ITEM(res, 2),
                                   writable ? Py_True : Py_False);
      if (ent) {
        PyDict_SetItem(self->cache, key, ent);
        Py_DECREF(ent);
      }
      Py_DECREF(ref);
    }
    PyErr_Clear(); /* objects that do not support weak references are simply not cached */
  }
  Py_DECREF(res);
  Py_DECREF(key);
  return 0;
}

static PyObject* running_loop(Binding* self) {
  PyObject* loop = PyObject_CallNoArgs(self->get_running_loop);
  if (!loop) return NULL;
  if (loop != self->last_loop) {
    PyObject* r = PyObject_CallOneArg(self->ensure_reader, loop);
    if (!r) {
      Py_DECREF(loop);
      return NULL;
    }
    Py_DECREF(r);
    Py_XDECREF(self->last_loop);
    Py_INCREF(loop);
    self->last_loop = loop;
  }
  return loop;
}

static PyObject* raise_last_error(Binding* self) {
  PyObject* msg = PyObject_CallNoArgs(self->last_error);
  if (msg) {
    PyErr_SetObject(PyExc_RuntimeError, msg);
    Py_DECREF(msg);
  }
  return NULL;
}

static PyObject* register_op(Binding* self, uint64_t op, PyObject* loop, PyObject* fut, PyObject* keep) {
  if (tab_insert(self, op, loop, fut, keep) < 0) {
    Py_DECREF(fut);
    return NULL;
  }
  return fut;
}

static PyObject* post_send_impl(Binding* self, uint64_t worker, uint64_t ep, PyObject* buffer, uint64_t tag) {
  void* ptr;
  size_t n;
  int mem;
  PyObject* keep;
  if (resolve_buffer(self, buffer, 0, &ptr, &n, &mem, &keep) < 0) return NULL;
  PyObject* loop = running_loop(self);
  PyObject* fut = loop ? PyObject_CallMethodNoArgs(loop, self->str_create_future) : NULL;
  if (!fut) {
    Py_XDECREF(loop);
    Py_DECREF(keep);
    return NULL;
  }
  /* the GIL is held from the post to the table insert: no other Python thread can observe the gap */
  uint64_t op = self->post_send(self->ctx, worker, ep, ptr, n, tag, mem);
  PyObject* ret = op ? register_op(self, op, loop, fut, keep) : (Py_DECREF(fut), raise_last_error(self));
  Py_DECREF(loop);
  Py_DECREF(keep);
  return ret;
}

static PyObject* post_recv_impl(Binding* self, uint64_t worker, PyObject* buffer, uint64_t tag, uint64_t mask) {
  void* ptr;
  size_t n;
  int mem;
  PyObject* keep;
  if (resolve_buffer(self, buffer, 1, &ptr, &n, &mem, &keep) < 0) return NULL;
  PyObject* loop = running_loop(self);
  PyObject* fut = loop ? PyObject_CallMethodNoArgs(loop, self->str_create_future) : NULL;
  if (!fut) {
    Py_XDECREF(loop);
    Py_DECREF(keep);
    return NULL;
  }
  uint64_t op = self->post_recv(self->ctx, worker, ptr, n, tag, mask, mem);
  PyObject* ret = op ? register_op(self, op, loop, fut, keep) : (Py_DECREF(fut), raise_last_error(self));
  Py_DECREF(loop);
  Py_DECREF(keep);
  return ret;
}

/* asend(worker, ep, buffer, tag) -> Future */
static PyObject* Binding_asend(Binding* self, PyObject* const* args, Py_ssize_t nargs) {
  if (nargs != 4) {
    PyErr_SetString(PyExc_TypeError, "asend(worker, ep, buffer, tag)");
    return NULL;
  }
  uint64_t worker = PyLong_AsUnsignedLongLong(args[0]);
  uint64_t ep = PyLong_AsUnsignedLongLong(args[1]);
  uint64_t tag = PyLong_AsUnsignedLongLongMask(args[3]);
  if (PyErr_Occurred()) return NULL;
  return post_send_impl(self, worker, ep, args[2], tag);
}

/* arecv(worker, buffer, tag, mask) -> Future */
static PyObject* Binding_arecv(Binding* self, PyObject* const* args, Py_ssize_t nargs) {
  if (nargs != 4) {
    PyErr_SetString(PyExc_TypeError, "arecv(worker, buffer, tag, tag_mask)");
    return NULL;
  }
  uint64_t worker = PyLong_AsUnsignedLongLong(args[0]);
  uint64_t tag = PyLong_AsUnsignedLongLongMask(args[2]);
  uint64_t mask = PyLong_AsUnsignedLongLongMask(args[3]);
  if (PyErr_Occurred()) return NULL;
  return post_recv_impl(self, worker, args[1], tag, mask);
}

/* ---- Post: `Client.asend` / `Client.arecv` / `Server.arecv` of one worker as a C callable.
 * The Python method did three attribute look-ups, a call into Binding.asend and a test of the polling state per
 * message; bound once per object, the call goes straight to the post.  Any call shape other than the common one
 * (an explicit loop, keywords) is handed to `slow`, the Python method it stands in for. */
typedef struct {
  PyObject_HEAD
  vectorcallfunc vc;
  Binding* b;
  PyObject* slow;
  uint64_t worker, ep;
  int is_recv;
} Post;

static PyObject* Post_call(PyObject* o, PyObject* const* args, size_t nargsf, PyObject* kwnames) {
  Post* p = (Post*)o;
  Py_ssize_t nargs = PyVectorcall_NARGS(nargsf);
  const Py_ssize_t want = p->is_recv ? 3 : 2;
  if (p->b->closed || (kwnames && PyTuple_GET_SIZE(kwnames)) || nargs < want || nargs > want + 1 || (nargs == want + 1 && args[want] != Py_None))
    return PyObject_Vectorcall(p->slow, args, nargsf & ~PY_VECTORCALL_ARGUMENTS_OFFSET, kwnames);
  PyObject* fut;
  if (p->is_recv) {
    uint64_t tag = PyLong_AsUnsignedLongLongMask(args[1]);
    uint64_t mask = PyLong_AsUnsignedLongLongMask(args[2]);
    if (PyErr_Occurred()) return NULL;
    fut = post_recv_impl(p->b, p->worker, args[0], tag, mask);
  } else {
    uint64_t tag = PyLong_AsUnsignedLongLongMask(args[1]);
    if (PyErr_Occurred()) return NULL;
    fut = post_send_impl(p->b, p->worker, p->ep, args[0], tag);
  }
  if (fut && !p->b->spinning && p->b->kick && p->b->kick != Py_None) {
    PyObject* r = PyObject_CallNoArgs(p->b->kick);
    if (!r) {
      Py_DECREF(fut);
      return NULL;
    }
    Py_DECREF(r);
  }
  return fut;
}

static void Post_dealloc(Post* p) {
  Py_XDECREF((PyObject*)p->b);
  Py_XDECREF(p->slow);
  Py_TYPE(p)->tp_free((PyObject*)p);
}

static PyTypeObject PostType = {
    PyVarObject_HEAD_INIT(NULL, 0).tp_name = "starway_b200._fastpath.Post",
    .tp_basicsize = sizeof(Post),
    .tp_flags = Py_TPFLAGS_DEFAULT | Py_TPFLAGS_HAVE_VECTORCALL,
    .tp_vectorcall_offset = offsetof(Post, vc),
    .tp_call = PyVectorcall_Call,
    .tp_dealloc = (destructor)Post_dealloc,
};

/* bound(worker, ep, is_recv, slow) -> Post */
static PyObject* Binding_bound(Binding* self, PyObject* args) {
  unsigned long long worker, ep;
  int is_recv;
  PyObject* slow;
  if (!PyArg_ParseTuple(args, "KKpO", &worker, &ep, &is_recv, &slow)) return NULL;
  Post* p = PyObject_New(Post, &PostType);
  if (!p) return NULL;
  p->vc = Post_call;
  Py_INCREF(self);
  p->b = self;
  Py_INCREF(slow);
  p->slow = slow;
  p->worker = worker;
  p->ep = ep;
  p->is_recv = is_recv;
  return (PyObject*)p;
}

static void swallow_invalid_state(void) {
  /* a future cancelled by the caller (asyncio.wait_for timeout ...) refuses the result: ignore */
  if (PyErr_Occurred()) PyErr_Clear();
}

/* set the result / exception of a future that belongs to the loop we are running on */
static int resolve_future(Binding* self, PyObject* fut, const sw_completion* c) {
  PyObject* r = NULL;
  if (c->status == 0) {
    if (c->kind == SW_OP_RECV) {
      PyObject* val = Py_BuildValue("(KK)", (unsigned long long)c->sender_tag, (unsigned long long)c->length);
      if (val) {
        r = PyObject_CallMethodOneArg(fut, self->str_set_result, val);
        Py_DECREF(val);
      }
    } else {
      r = PyObject_CallMethodOneArg(fut, self->str_set_result, Py_None);
    }
  } else {
    PyObject* msg = PyObject_CallFunction(self->status_string, "i", (int)c->status);
    PyObject* exc = msg ? PyObject_CallOneArg(PyExc_Exception, msg) : NULL;
    if (exc) r = PyObject_CallMethodOneArg(fut, self->str_set_exception, exc);
    Py_XDECREF(msg);
    Py_XDECREF(exc);
  }
  if (!r) swallow_invalid_state();
  Py_XDECREF(r);
  return 0;
}

/* A Python error raised while one completion is handed over (user callback, hand-over to another
 * loop) is reported and the batch goes on: the completions already polled belong to other operations. */
static void report_and_continue(Binding* self) {
  if (PyErr_Occurred()) PyErr_WriteUnraisable((PyObject*)self);
}

/* drain(loop): resolve every pending completion; runs on `loop`'s thread (eventfd reader) */
static PyObject* Binding_drain(Binding* self, PyObject* here) {
  /* the batch lives on this thread's stack: resolving an entry may run Python code (the shim), which
   * can release the GIL and let another loop's thread enter drain() on the same Binding */
  enum { BATCH = 256 };
  sw_completion batch[BATCH];
  long total = 0;
  for (;;) {
    int n = self->poll(self->ctx, batch, BATCH);
    if (n <= 0) break;
    total += n;
    for (int i = 0; i < n; i++) {
      const sw_completion c = batch[i];
      OpSlot* slot = tab_find(self, c.op_id);
      if (slot) {
        PyObject *loop = slot->loop, *fut = slot->fut, *keep = slot->keep; /* references move to us */
        tab_remove(self, slot);
        int rc = 0;
        if (loop == here) {
          rc = resolve_future(self, fut, &c);
        } else {
          /* a future of another loop: the Python shim hands it over with call_soon_threadsafe */
          PyObject* entry = PyTuple_Pack(5, self->str_fut, loop, fut, keep, Py_None);
          PyObject* r = entry ? PyObject_CallFunction(self->slow, "OIiKKKKOK", entry, (unsigned)c.kind, (int)c.status,
                                                      (unsigned long long)c.sender_tag, (unsigned long long)c.length,
                                                      (unsigned long long)c.worker, (unsigned long long)c.ep, here,
                                                      (unsigned long long)c.op_id)
                              : NULL;
          if (!r) rc = -1;
          Py_XDECREF(r);
          Py_XDECREF(entry);
        }
        Py_DECREF(loop);
        Py_DECREF(fut);
        Py_DECREF(keep);
        if (rc < 0) report_and_continue(self); /* one failing hand-over must not drop the rest of the batch */
        continue;
      }
      /* not a fast-path operation: the table shared with the Python shim */
      PyObject* key = PyLong_FromUnsignedLongLong(c.op_id);
      if (!key) {
        report_and_continue(self);
        continue;
      }
      PyObject* entry = PyDict_GetItemWithError(self->ops, key); /* borrowed */
      if (entry) {
        Py_INCREF(entry);
        PyDict_DelItem(self->ops, key);
      } else if (PyErr_Occurred()) {
        report_and_continue(self);
      }
      Py_DECREF(key);
      int fast = entry && PyTuple_Check(entry) && PyTuple_GET_SIZE(entry) == 5 &&
                 PyTuple_GET_ITEM(entry, 0) == self->str_fut && PyTuple_GET_ITEM(entry, 1) == here &&
                 PyTuple_GET_ITEM(entry, 4) == Py_None;
      if (fast) {
        if (resolve_future(self, PyTuple_GET_ITEM(entry, 2), &c) < 0) report_and_continue(self);
      } else {
        /* accept notifications, raw callbacks, other loops, banner callbacks -- and operations another
         * thread posted through the ctypes path (GIL released inside sw_post_*) but has not registered
         * yet: the Python shim looks those up again under the context lock (op id passed along) */
        PyObject* r = PyObject_CallFunction(self->slow, "OIiKKKKOK", entry ? entry : Py_None, (unsigned)c.kind, (int)c.status,
                                            (unsigned long long)c.sender_tag, (unsigned long long)c.length,
                                            (unsigned long long)c.worker, (unsigned long long)c.ep, here,
                                            (unsigned long long)c.op_id);
        if (!r) report_and_continue(self);
        Py_XDECREF(r);
      }
      Py_XDECREF(entry);
    }
    if (n < BATCH) break;
  }
  return PyLong_FromLong(total);
}

/* take(op_id) -> ("fut", loop, fut, keep, None) | None: hands a fast-path entry to the Python shim
 * (completions polled by the fallback poller thread instead of a loop's reader) */
static PyObject* Binding_take(Binding* self, PyObject* arg) {
  uint64_t op = PyLong_AsUnsignedLongLong(arg);
  if (PyErr_Occurred()) return NULL;
  OpSlot* slot = tab_find(self, op);
  if (!slot) Py_RETURN_NONE;
  PyObject *loop = slot->loop, *fut = slot->fut, *keep = slot->keep;
  tab_remove(self, slot);
  PyObject* entry = PyTuple_Pack(5, self->str_fut, loop, fut, keep, Py_None);
  Py_DECREF(loop);
  Py_DECREF(fut);
  Py_DECREF(keep);
  return entry;
}

static PyObject* Binding_pending(Binding* self, PyObject* Py_UNUSED(ignored)) {
  return PyLong_FromSize_t(self->tab_count);
}

static PyMethodDef Binding_methods[] = {
    {"take", (PyCFunction)Binding_take, METH_O, "take(op_id) -> entry tuple or None"},
    {"pending", (PyCFunction)Binding_pending, METH_NOARGS, "pending() -> int: fast-path operations awaiting completion"},
    {"asend", (PyCFunction)(void (*)(void))Binding_asend, METH_FASTCALL, "asend(worker, ep, buffer, tag) -> Future"},
    {"arecv", (PyCFunction)(void (*)(void))Binding_arecv, METH_FASTCALL, "arecv(worker, buffer, tag, mask) -> Future"},
    {"drain", (PyCFunction)Binding_drain, METH_O, "drain(loop) -> int: resolve pending completions on the loop thread"},
    {"bound", (PyCFunction)Binding_bound, METH_VARARGS, "bound(worker, ep, is_recv, slow) -> callable posting for that worker"},
    {NULL, NULL, 0, NULL}};

static PyMemberDef Binding_members[] = {
    {"kick", T_OBJECT, offsetof(Binding, kick), 0, "callable that starts completion polling on the running loop"},
    {"spinning", T_INT, offsetof(Binding, spinning), 0, "non-zero while the loop polls the completion queue"},
    {"closed", T_INT, offsetof(Binding, closed), 0, "non-zero once the context is being closed"},
    {NULL, 0, 0, 0, NULL}};

static PyTypeObject BindingType = {
    PyVarObject_HEAD_INIT(NULL, 0).tp_name = "starway_b200._fastpath.Binding",
    .tp_basicsize = sizeof(Binding),
    .tp_flags = Py_TPFLAGS_DEFAULT,
    .tp_new = PyType_GenericNew,
    .tp_init = (initproc)Binding_init,
    .tp_dealloc = (destructor)Binding_dealloc,
    .tp_methods = Binding_methods,
    .tp_members = Binding_members,
};

static struct PyModuleDef moddef = {PyModuleDef_HEAD_INIT, "_fastpath",
                                    "C fast path of the starway_b200 binding layer (post / poll / future resolution)", -1,
                                    NULL};

PyMODINIT_FUNC PyInit__fastpath(void) {
  if (PyType_Ready(&BindingType) < 0 || PyType_Ready(&PostType) < 0) return NULL;
  PyObject* m = PyModule_Create(&moddef);
  if (!m) return NULL;
  Py_INCREF(&BindingType);
  if (PyModule_AddObject(m, "Binding", (PyObject*)&BindingType) < 0) {
    Py_DECREF(&BindingType);
    Py_DECREF(m);
    return NULL;
  }
  return m;
}
