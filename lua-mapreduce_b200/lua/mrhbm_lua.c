/*
 * mrhbm_lua.c -- Lua 5.2 C module "mrhbm": the binding a lua-mapreduce maintainer adds so that
 * storage = "hbm" reaches the C ABI of include/mrhbm.h.  It takes the place luamongo has on the
 * reference's hot path (external/luamongo/mongo_gridfilebuilder.cpp:55-92 append/build,
 * mongo_gridfs.cpp:117-144 list, mongo_gridfile.cpp:38-59 chunk) and keeps its conventions:
 * every method returns `nil, "<msg>"` on failure and never throws into Lua; userdata are
 * released in __gc.
 *
 * NOT COMPILED IN THIS IMAGE (no lua.h): the exact same call sequence is exercised through
 * the ctypes binding lua-mapreduce_b200/mrhbm.py by tests/.  Build where Lua 5.2 exists:
 *   gcc -O2 -fPIC -shared -I/usr/include/lua5.2 -I../../include mrhbm_lua.c \
 *       -L../lib -lmrhbm -o mrhbm.so
 */
#include <lauxlib.h>
#include <lua.h>
#include <math.h>
#include <string.h>

#include "mrhbm.h"

#ifndef LUA_TSTRING
#define LUA_TSTRING 4 /* the same in lua.h of every Lua 5.x (for declaration-only builds of this file) */
#endif

#define CTX_MT "mrhbm.ctx"
#define MAP_MT "mrhbm.map"
#define ITER_MT "mrhbm.iter"

typedef struct { mrhbm_ctx *h; uint32_t nparts; int bytes; } lctx; /* bytes: values = "bytes" */
typedef struct { mrhbm_map *h; mrhbm_ctx *ctx; int bytes; } lmap;
typedef struct { mrhbm_iter *h; int bytes; } liter;

static int fail(lua_State *L, mrhbm_ctx *c) { /* luamongo style: nil, msg */
  lua_pushnil(L);
  lua_pushstring(L, c ? mrhbm_last_error(c) : "mrhbm: invalid handle");
  return 2;
}

/* mrhbm.new{ key_kind="str"|"u64", max_key_bytes=, num_partitions=, partitioner="fnv_lua"|"mulhash"|
 *            "wordhash"|"range", combiner=bool|"distinct"|"fsum", reducer="sum"|"none"|"distinct"|"fsum"|
 *            "count_distinct", device=, values="int"|"bytes" }
 * values = "bytes" (MRHBM_F_BYTE_VALUES, needs reducer = "none", "distinct", "fsum" or "count_distinct"): m:emit takes
 * string values and ctx:groups yields tables of strings (reducer = "distinct": each key's distinct values, ascending;
 * reducer = "fsum": one value, the exact sum of the key's numbers; reducer = "count_distinct": one value, the number
 * of the key's distinct values) */
static int l_new(lua_State *L) {
  mrhbm_config cfg;
  const char *s;
  memset(&cfg, 0, sizeof cfg);
  cfg.struct_size = sizeof cfg;
  luaL_checktype(L, 1, LUA_TTABLE);
  lua_getfield(L, 1, "key_kind");
  s = luaL_optstring(L, -1, "str");
  cfg.key_kind = strcmp(s, "u64") == 0 ? MRHBM_KEY_U64 : MRHBM_KEY_STR;
  lua_getfield(L, 1, "max_key_bytes");
  cfg.max_key_bytes = (uint32_t)luaL_optinteger(L, -1, 123);
  lua_getfield(L, 1, "num_partitions");
  cfg.num_partitions = (uint32_t)luaL_checkinteger(L, -1);
  lua_getfield(L, 1, "partitioner");
  s = luaL_optstring(L, -1, cfg.key_kind == MRHBM_KEY_U64 ? "mulhash" : "fnv_lua");
  cfg.partitioner = strcmp(s, "fnv_lua") == 0 ? MRHBM_PART_FNV_LUA
                  : strcmp(s, "mulhash") == 0 ? MRHBM_PART_MULHASH
                  : strcmp(s, "range") == 0 ? MRHBM_PART_RANGE : MRHBM_PART_WORDHASH;
  lua_getfield(L, 1, "combiner"); /* true (the built-in reducer) | "distinct" | "fsum" (values = "bytes") */
  cfg.combiner = lua_type(L, -1) == LUA_TSTRING && strcmp(luaL_checkstring(L, -1), "distinct") == 0 ? MRHBM_COMBINE_DISTINCT
               : lua_type(L, -1) == LUA_TSTRING && strcmp(luaL_checkstring(L, -1), "fsum") == 0   ? MRHBM_COMBINE_FSUM
               : lua_toboolean(L, -1) ? MRHBM_COMBINE_REDUCER : MRHBM_COMBINE_NONE;
  lua_getfield(L, 1, "device");
  cfg.device = (int32_t)luaL_optinteger(L, -1, -1);
  lua_getfield(L, 1, "reducer"); /* "sum" (built-in) | "none" (general reducefn on the host) | "distinct" | "fsum" |
                                    "count_distinct" */
  s = luaL_optstring(L, -1, "sum");
  cfg.reducer = strcmp(s, "none") == 0             ? MRHBM_RED_NONE
                : strcmp(s, "distinct") == 0       ? MRHBM_RED_DISTINCT
                : strcmp(s, "fsum") == 0           ? MRHBM_RED_FSUM
                : strcmp(s, "count_distinct") == 0 ? MRHBM_RED_COUNT_DISTINCT
                                                   : MRHBM_RED_SUM;
  lua_getfield(L, 1, "values");
  s = luaL_optstring(L, -1, "int");
  if (strcmp(s, "bytes") == 0) cfg.flags |= MRHBM_F_BYTE_VALUES;
  lua_pop(L, 8);
  lctx *u = (lctx *)lua_newuserdata(L, sizeof *u);
  u->h = NULL;
  u->nparts = cfg.num_partitions;
  u->bytes = (cfg.flags & MRHBM_F_BYTE_VALUES) != 0;
  luaL_setmetatable(L, CTX_MT);
  if (mrhbm_init(&cfg, &u->h) != MRHBM_OK) {
    lua_pushnil(L);
    lua_pushstring(L, u->h ? mrhbm_last_error(u->h) : "mrhbm_init failed");
    if (u->h) mrhbm_destroy(u->h);
    u->h = NULL;
    return 2;
  }
  return 1;
}
static lctx *checkctx(lua_State *L) { return (lctx *)luaL_checkudata(L, 1, CTX_MT); }
static int ctx_gc(lua_State *L) {
  lctx *u = checkctx(L);
  if (u->h) mrhbm_destroy(u->h);
  u->h = NULL;
  return 0;
}
/* ctx:map_begin(job_id) -> map  (job.lua:83-97: the emit buffer of one map job) */
static int ctx_map_begin(lua_State *L) {
  lctx *u = checkctx(L);
  const char *id = luaL_checkstring(L, 2);
  lmap *m = (lmap *)lua_newuserdata(L, sizeof *m);
  m->h = NULL;
  m->ctx = u->h;
  m->bytes = u->bytes;
  luaL_setmetatable(L, MAP_MT);
  /* the map keeps its ctx alive (Lua 5.2 user values are tables): commit / abort / __gc dereference it */
  lua_createtable(L, 1, 0);
  lua_pushvalue(L, 1);
  lua_rawseti(L, -2, 1);
  lua_setuservalue(L, -2);
  if (mrhbm_map_begin(u->h, id, &m->h) != MRHBM_OK) return fail(L, u->h);
  return 1;
}
/* map:emit(key, value) with values = "bytes": value is a Lua string (any bytes, copied before return) */
static int map_emit_bytes(lua_State *L, lmap *m, int u64) {
  size_t vlen, len;
  const char *v = luaL_checklstring(L, 3, &vlen);
  int rc;
  if (lua_type(L, 2) == LUA_TNUMBER) {
    lua_Number kn = lua_tonumber(L, 2);
    if (!u64 || !(kn >= 0 && kn == floor(kn) && kn < 9007199254740992.0)) {
      lua_pushnil(L);
      lua_pushstring(L, "mrhbm: number keys need key_kind = 'u64' and an integer in [0, 2^53)");
      return 2;
    }
    rc = mrhbm_emit_u64_value(m->h, (uint64_t)kn, v, vlen);
  } else {
    const char *k = luaL_checklstring(L, 2, &len);
    if (u64 && len == 8) {
      uint64_t x = 0;
      for (int i = 0; i < 8; i++) x = (x << 8) | (unsigned char)k[i];
      rc = mrhbm_emit_u64_value(m->h, x, v, vlen);
    } else
      rc = mrhbm_emit_str_value(m->h, k, len, v, vlen);
  }
  if (rc != MRHBM_OK) return fail(L, m->ctx);
  lua_pushboolean(L, 1);
  return 1;
}
/* map:emit(key, value): key is a Lua string (copied before return) or, for u64 ctx, an 8-byte
 * big-endian string / an integer-valued number < 2^53 (SURVEY A.4) */
static int map_emit(lua_State *L) {
  lmap *m = (lmap *)luaL_checkudata(L, 1, MAP_MT);
  int rc;
  int u64 = m->h && mrhbm_record_bytes(m->ctx) == 16;
  if (!m->h) return fail(L, NULL);
  if (m->bytes) return map_emit_bytes(L, m, u64);
  lua_Number vn = luaL_optnumber(L, 3, 1);
  /* values are unsigned integers: < 2^32 in string records, < 2^53 (exact Lua numbers) with u64 keys.  Anything
   * else is refused here -- a C cast of an out-of-range double is undefined behaviour, not a wrap-around. */
  if (!(vn >= 0 && vn == floor(vn) && vn < (u64 ? 9007199254740992.0 : 4294967296.0))) {
    lua_pushnil(L);
    lua_pushstring(L, u64 ? "mrhbm: value must be an integer in [0, 2^53)" : "mrhbm: value must be an integer in [0, 2^32)");
    return 2;
  }
  uint64_t v = (uint64_t)vn;
  if (lua_type(L, 2) == LUA_TNUMBER) {
    lua_Number kn = lua_tonumber(L, 2);
    if (!u64 || !(kn >= 0 && kn == floor(kn) && kn < 9007199254740992.0)) {
      lua_pushnil(L);
      lua_pushstring(L, "mrhbm: number keys need key_kind = 'u64' and an integer in [0, 2^53)");
      return 2;
    }
    rc = mrhbm_emit_u64(m->h, (uint64_t)kn, v);
  } else {
    size_t len;
    const char *k = luaL_checklstring(L, 2, &len);
    if (u64 && len == 8) {
      uint64_t x = 0;
      for (int i = 0; i < 8; i++) x = (x << 8) | (unsigned char)k[i];
      rc = mrhbm_emit_u64(m->h, x, v);
    } else
      rc = mrhbm_emit_str(m->h, k, len, (uint32_t)v);
  }
  if (rc != MRHBM_OK) return fail(L, m->ctx);
  lua_pushboolean(L, 1);
  return 1;
}
/* map:wordcount(text) -> number of words: the WordCount mapfn on the device
 * (examples/WordCount/mapfn.lua:3-9), text is one Lua string (e.g. a whole file) */
static int map_wordcount(lua_State *L) {
  lmap *m = (lmap *)luaL_checkudata(L, 1, MAP_MT);
  size_t len;
  const char *t = luaL_checklstring(L, 2, &len);
  uint64_t n = 0;
  if (!m->h || mrhbm_map_wordcount(m->h, t, len, &n) != MRHBM_OK) return fail(L, m->ctx);
  lua_pushnumber(L, (lua_Number)n);
  return 1;
}
/* map:words_value(text, value) -> number of words, with values = "bytes": the same tokeniser emitting (word, value)
 * for every word (an inverted index's mapfn), value is a Lua string (copied before return) */
static int map_words_value(lua_State *L) {
  lmap *m = (lmap *)luaL_checkudata(L, 1, MAP_MT);
  size_t len, vlen;
  const char *t = luaL_checklstring(L, 2, &len);
  const char *v = luaL_checklstring(L, 3, &vlen);
  uint64_t n = 0;
  if (!m->h || mrhbm_map_words_value(m->h, t, len, v, vlen, &n) != MRHBM_OK) return fail(L, m->ctx);
  lua_pushnumber(L, (lua_Number)n);
  return 1;
}
/* map:key_numbers(text) -> number of pairs, with values = "bytes" and string keys: every line "key number" of the
 * text becomes (key, the number's value encoding), parsed on the device (a number sum's mapfn) */
static int map_key_numbers(lua_State *L) {
  lmap *m = (lmap *)luaL_checkudata(L, 1, MAP_MT);
  size_t len;
  const char *t = luaL_checklstring(L, 2, &len);
  uint64_t n = 0;
  if (!m->h || mrhbm_map_key_numbers(m->h, t, len, &n) != MRHBM_OK) return fail(L, m->ctx);
  lua_pushnumber(L, (lua_Number)n);
  return 1;
}
static int map_commit(lua_State *L) { /* job.lua:217-221: remove_file + build */
  lmap *m = (lmap *)luaL_checkudata(L, 1, MAP_MT);
  mrhbm_map *h = m->h;
  m->h = NULL;
  if (!h || mrhbm_map_commit(h) != MRHBM_OK) return fail(L, m->ctx);
  lua_pushboolean(L, 1);
  return 1;
}
static int map_abort(lua_State *L) { /* worker.lua:120-127 and __gc */
  lmap *m = (lmap *)luaL_checkudata(L, 1, MAP_MT);
  if (m->h) mrhbm_map_abort(m->h);
  m->h = NULL;
  return 0;
}
static int ctx_shuffle(lua_State *L) { /* server.lua:279-329 barrier */
  lctx *u = checkctx(L);
  if (mrhbm_shuffle(u->h) != MRHBM_OK) return fail(L, u->h);
  lua_pushboolean(L, 1);
  return 1;
}
static int ctx_reset(lua_State *L) {
  lctx *u = checkctx(L);
  if (mrhbm_reset(u->h) != MRHBM_OK) return fail(L, u->h);
  lua_pushboolean(L, 1);
  return 1;
}
static int ctx_partitions(lua_State *L) { /* server.lua:300-324: one reduce job per non-empty partition */
  lctx *u = checkctx(L);
  size_t n = 0, i;
  if (mrhbm_partitions(u->h, NULL, 0, &n) != MRHBM_OK) return fail(L, u->h);
  uint32_t *ids = (uint32_t *)lua_newuserdata(L, (n ? n : 1) * sizeof *ids);
  mrhbm_partitions(u->h, ids, n, &n);
  lua_createtable(L, (int)n, 0);
  for (i = 0; i < n; i++) {
    lua_pushinteger(L, ids[i]);
    lua_rawseti(L, -2, (int)i + 1);
  }
  return 1;
}
/* ctx:set_splitters(s_0, s_1, ..., s_{P-2}) -> true  (range partitioner: the splitters as strings, u64 keys as
 * their 8 big-endian bytes; mapreduce/hbm.lua passes a table's elements with table.unpack) */
static int ctx_set_splitters(lua_State *L) {
  lctx *u = checkctx(L);
  size_t n = 0, total = 0, len, i;
  while (lua_type(L, (int)n + 2) > 0) { /* LUA_TNONE = -1 past the last argument, LUA_TNIL = 0 */
    luaL_checklstring(L, (int)n + 2, &len);
    total += len;
    n++;
  }
  char *keys = (char *)lua_newuserdata(L, total ? total : 1);
  uint64_t *off = (uint64_t *)lua_newuserdata(L, (n + 1) * sizeof(uint64_t));
  off[0] = 0;
  for (i = 0; i < n; i++) {
    const char *k = luaL_checklstring(L, (int)i + 2, &len);
    memcpy(keys + off[i], k, len);
    off[i + 1] = off[i] + len;
  }
  if (mrhbm_set_splitters(u->h, keys, off, n) != MRHBM_OK) return fail(L, u->h);
  lua_pushboolean(L, 1);
  return 1;
}
/* ctx:sample_splitters() -> { s_0, ..., s_{P-2} }  (range partitioner: quantiles of a sample of the committed pairs,
 * installed; collective on several GPUs) */
static int ctx_sample_splitters(lua_State *L) {
  lctx *u = checkctx(L);
  size_t need = 0, n = u->nparts ? u->nparts - 1 : 0, i;
  uint32_t rb = u->h ? mrhbm_record_bytes(u->h) : 16;
  size_t cap = n * (rb == 16 ? 8 : rb - 4) + 1; /* a splitter takes at most one key slot: one call, no sizing call */
  uint64_t *off = (uint64_t *)lua_newuserdata(L, (n + 1) * sizeof(uint64_t));
  char *keys = (char *)lua_newuserdata(L, cap);
  if (mrhbm_sample_splitters(u->h, keys, cap, off, &need) != MRHBM_OK) return fail(L, u->h);
  lua_createtable(L, (int)n, 0);
  for (i = 0; i < n; i++) {
    lua_pushlstring(L, keys + off[i], (size_t)(off[i + 1] - off[i]));
    lua_rawseti(L, -2, (int)i + 1);
  }
  return 1;
}
/* ctx:groups(partition) -> iterator yielding key, values  (utils.merge_iterator's consumer,
 * job.lua:264-284; also finalfn's pair iterator, server.lua:360-385) */
static int iter_next(lua_State *L) {
  liter *it = (liter *)lua_touserdata(L, lua_upvalueindex(1));
  const void *key, *bytes = NULL;
  const uint64_t *vals = NULL, *voff = NULL;
  size_t klen, nvals, i;
  int r = !it->h ? 0
        : it->bytes ? mrhbm_groups_next_values(it->h, &key, &klen, &bytes, &voff, &nvals)
                    : mrhbm_groups_next(it->h, &key, &klen, &vals, &nvals);
  if (r <= 0) {
    if (it->h) mrhbm_groups_close(it->h);
    it->h = NULL;
    return 0;
  }
  lua_pushlstring(L, (const char *)key, klen);
  lua_createtable(L, (int)nvals, 0);
  for (i = 0; i < nvals; i++) {
    if (it->bytes)
      lua_pushlstring(L, (const char *)bytes + voff[i], (size_t)(voff[i + 1] - voff[i]));
    else
      lua_pushnumber(L, (lua_Number)vals[i]); /* sums < 2^53 are exact Lua numbers */
    lua_rawseti(L, -2, (int)i + 1);
  }
  return 2;
}
static int iter_gc(lua_State *L) {
  liter *it = (liter *)luaL_checkudata(L, 1, ITER_MT);
  if (it->h) mrhbm_groups_close(it->h);
  it->h = NULL;
  return 0;
}
static int ctx_groups(lua_State *L) {
  lctx *u = checkctx(L);
  uint32_t p = (uint32_t)luaL_checkinteger(L, 2);
  liter *it = (liter *)lua_newuserdata(L, sizeof *it);
  it->h = NULL;
  it->bytes = u->bytes;
  luaL_setmetatable(L, ITER_MT);
  if (mrhbm_groups_open(u->h, p, &it->h) != MRHBM_OK) return fail(L, u->h);
  lua_pushvalue(L, 1); /* second upvalue: the ctx stays alive as long as the iterator function does */
  lua_pushcclosure(L, iter_next, 2);
  return 1;
}

static const luaL_Reg ctx_methods[] = {{"map_begin", ctx_map_begin}, {"shuffle", ctx_shuffle},
                                       {"partitions", ctx_partitions}, {"groups", ctx_groups},
                                       {"reset", ctx_reset}, {"set_splitters", ctx_set_splitters},
                                       {"sample_splitters", ctx_sample_splitters}, {"__gc", ctx_gc}, {NULL, NULL}};
static const luaL_Reg map_methods[] = {{"emit", map_emit}, {"wordcount", map_wordcount},
                                       {"words_value", map_words_value}, {"key_numbers", map_key_numbers}, {"commit", map_commit},
                                       {"abort", map_abort}, {"__gc", map_abort}, {NULL, NULL}};
static const luaL_Reg mod_funcs[] = {{"new", l_new}, {NULL, NULL}};

int luaopen_mrhbm(lua_State *L) {
  luaL_newmetatable(L, CTX_MT);
  lua_pushvalue(L, -1);
  lua_setfield(L, -2, "__index");
  luaL_setfuncs(L, ctx_methods, 0);
  luaL_newmetatable(L, MAP_MT);
  lua_pushvalue(L, -1);
  lua_setfield(L, -2, "__index");
  luaL_setfuncs(L, map_methods, 0);
  luaL_newmetatable(L, ITER_MT);
  lua_pushcfunction(L, iter_gc);
  lua_setfield(L, -2, "__gc");
  lua_pop(L, 3);
  luaL_newlib(L, mod_funcs);
  lua_pushinteger(L, MRHBM_ABI_VERSION);
  lua_setfield(L, -2, "_ABI");
  return 1;
}
