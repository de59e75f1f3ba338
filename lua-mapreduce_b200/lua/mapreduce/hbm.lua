-- mapreduce/hbm.lua -- the "hbm" storage of lua-mapreduce: replaces the text spill through
-- GridFS / shared FS / scp (mapreduce/fs.lua:185-208) by the in-HBM shuffle of the mrhbm C
-- module.  The seam sits one level above fs.router: job.lua's emit closure (job.lua:83-97) and
-- the consumer of utils.merge_iterator (job.lua:264-284) call this module, so no "%q" line is
-- ever formatted or load()-ed.
--
-- NOT EXECUTABLE IN THE BUILD IMAGE (no Lua).  The Python mirror in ../../mapreduce/ runs
-- the same call sequence against the same C ABI under test.
local mrhbm = require "mrhbm"

local hbm = { _VERSION = "0.1", _NAME = "mapreduce.hbm" }

-- what the device evaluates is declared on the plugin tables, like the reducer algebra flags
-- (examples/WordCount/reducefn.lua:10-14):
--   partitionfn module: hbm_partitionfn = "fnv_lua" | "wordhash" | "mulhash", NUM_REDUCERS = n
--     or a key range: hbm_partitionfn = "range", hbm_splitters = { s_1, ..., s_{n-1} } (non-decreasing strings; u64
--     keys as their 8 big-endian bytes; partition k takes the keys k splitters are <= to) or hbm_splitters = "sample"
--     (quantiles of the map output, taken at the MAP -> REDUCE barrier).  The partitionfn must compute the same ranges.
--   reducefn / combinerfn module: hbm_reducefn = "sum"; a combinerfn module of a value_kind = "bytes" job:
--     hbm_combinerfn = "distinct" (its combinerfn emits the distinct values it is given), or, with hbm_reducefn =
--     "fsum", hbm_combinerfn = "fsum" (its combinerfn emits the sum of its number values; the device keeps each map
--     job's sum per key exactly, as one or two numbers, so the result is the reducer's alone); a reducefn module of a
--     value_kind = "bytes" job: hbm_reducefn = "fsum" (its reducefn emits the sum of its number values; the device
--     sums them exactly, rounds once, and hbm.groups hands out that one number), or hbm_reducefn = "distinct" (its
--     reducefn emits the distinct values ascending by their
--     encoded bytes; the device computes them and hbm.groups hands them out as the reducefn's result), or
--     hbm_reducefn = "count_distinct" (its reducefn emits the number of distinct values, a table used as a set then
--     emit(n); the device counts them by their encoded bytes and hbm.groups hands out that one number)
local ctx -- one context per worker process (job.lua keeps `funcs`/`initialized` per process too)
local sample_splitters = false -- hbm_splitters = "sample": hbm.prepare_reduce samples them before the shuffle
local tuple_keys = false -- hbm.configure(..., { key_kind = "tuple" }); an upvalue of configure, map_job and groups
local byte_values = false -- hbm.configure(..., { value_kind = "bytes" }): string and number values, general reducefn

-- the 8-byte big-endian string of a u64 key minus one; nil for key 0
local function be_minus_one(s)
  local b = { s:byte(1, #s) }
  local i = #b
  while i >= 1 and b[i] == 0 do
    b[i] = 255
    i = i - 1
  end
  if i < 1 then return nil end
  b[i] = b[i] - 1
  return string.char(table.unpack(b))
end

function hbm.configure(partition_mod, reduce_mod, combiner_mod, opts)
  -- hbm_reducefn = "sum": reduced on the device.  No declaration: general reducer -- the device
  -- partitions, sorts and groups, job.lua:264-284 calls reducefn per group on the host.
  local builtin = reduce_mod.hbm_reducefn == "sum"
  local distinct_red = reduce_mod.hbm_reducefn == "distinct"
  local fsum_red = reduce_mod.hbm_reducefn == "fsum"
  local count_red = reduce_mod.hbm_reducefn == "count_distinct"
  opts = opts or {}
  tuple_keys = opts.key_kind == "tuple" -- composite keys travel as encoded byte strings
  byte_values = opts.value_kind == "bytes" -- values travel as encoded byte strings (hbm.encode_value)
  assert(not (byte_values and reduce_mod.hbm_reducefn ~= nil and not distinct_red and not fsum_red and not count_red),
         "value_kind = 'bytes' hands string and number values to a general reducefn: the reducefn must not declare an hbm_reducefn other than 'distinct', 'fsum' or 'count_distinct'")
  assert(not distinct_red or byte_values, "hbm_reducefn = 'distinct' needs value_kind = 'bytes'")
  assert(not fsum_red or byte_values, "hbm_reducefn = 'fsum' needs value_kind = 'bytes'")
  assert(not count_red or byte_values, "hbm_reducefn = 'count_distinct' needs value_kind = 'bytes'")
  -- hbm_combinerfn = "fsum" (hbm_reducefn = "fsum"): each map job's numbers per key become the exact expansion of
  -- their sum at its commit (include/mrhbm.h, MRHBM_COMBINE_FSUM)
  local fsum_comb = combiner_mod ~= nil and combiner_mod.hbm_combinerfn == "fsum"
  assert(not fsum_comb or fsum_red, "hbm_combinerfn = 'fsum' needs hbm_reducefn = 'fsum' and value_kind = 'bytes'")
  assert(not fsum_red or combiner_mod == nil or fsum_comb, "hbm_reducefn = 'fsum' takes no combinerfn but hbm_combinerfn = 'fsum'")
  -- hbm_combinerfn = "distinct" (values = "bytes"): the combinerfn keeps one copy of each distinct value of a key, so
  -- the device drops the repeated (key, value) pairs of each map job at its commit
  local distinct = combiner_mod ~= nil and combiner_mod.hbm_combinerfn == "distinct"
  assert(not distinct or byte_values, "hbm_combinerfn = 'distinct' needs value_kind = 'bytes'")
  assert(not combiner_mod or distinct or fsum_comb or (builtin and combiner_mod.hbm_reducefn == "sum"),
         "a combinerfn runs on the device: it (and the reducefn) must declare hbm_reducefn = 'sum', or hbm_combinerfn = 'distinct' or 'fsum' with value_kind = 'bytes'")
  local c, err = mrhbm.new{
    key_kind = tuple_keys and "str" or opts.key_kind or "str",
    max_key_bytes = opts.max_key_bytes or 123,
    num_partitions = assert(partition_mod.NUM_REDUCERS, "partitionfn module must expose NUM_REDUCERS"),
    partitioner = assert(partition_mod.hbm_partitionfn, "partitionfn module must declare hbm_partitionfn"),
    combiner = distinct and "distinct" or (fsum_comb and "fsum" or combiner_mod ~= nil),
    reducer = builtin and "sum" or (distinct_red and "distinct" or (fsum_red and "fsum" or
              (count_red and "count_distinct" or "none"))),
    device = opts.device,
    values = byte_values and "bytes" or "int",
  }
  ctx = assert(c, err)
  sample_splitters = false
  if partition_mod.hbm_partitionfn == "range" then
    local spl = partition_mod.hbm_splitters
    if spl == "sample" then
      sample_splitters = true
    else
      assert(type(spl) == "table", "hbm_partitionfn = 'range' needs hbm_splitters = {...} or 'sample'")
      assert(#spl + 1 == partition_mod.NUM_REDUCERS, "NUM_REDUCERS must equal the number of splitters + 1")
      local u64 = opts.key_kind == "u64" -- u64 keys: 8-byte big-endian strings
      for i = 1, #spl do
        assert(not u64 or #spl[i] == 8, "u64 splitters are 8-byte big-endian strings")
        assert(i == 1 or not (spl[i] < spl[i - 1]), "hbm_splitters must be non-decreasing")
      end
      -- the declaration must describe the same key ranges as partitionfn: the key of splitter i goes above every
      -- splitter equal to it (bisect_right), and for u64 keys the key just below it goes below them
      for i = 1, #spl do
        local j = i
        while spl[j + 1] == spl[i] do j = j + 1 end
        assert(partition_mod.partitionfn(spl[i]) == j, "partitionfn disagrees with hbm_splitters at " .. spl[i])
        local below = u64 and be_minus_one(spl[i])
        if below then
          local k = i - 1
          while k >= 1 and not (spl[k] <= below) do k = k - 1 end
          assert(partition_mod.partitionfn(below) == k, "partitionfn disagrees with hbm_splitters just below " .. spl[i])
        end
      end
      assert(ctx:set_splitters(table.unpack(spl)))
    end
  end
  return ctx
end


-- ---------------------------------------------------------------------------------------------
-- Composite keys (mapreduce/tuple.lua): a tuple key crosses the C ABI as an ORDER-PRESERVING,
-- NUL-free byte string (<= 123 bytes) and is decoded again on the reduce side.  Same format as
-- ../../mapreduce/tuple.py (which is what runs under test):
--   key       := "\127" component | char(128+n) component*n       (n <= 31, shorter tuples first)
--   component := "\16" num10 | "\32" bytes "\1" | "\48" key
--   num10     := the IEEE double, sign-folded so that unsigned order = numeric order, as 10
--                big-endian 7-bit groups each OR 0x80
-- Bytewise order = length first, then component-wise: a linear extension of tuple.lua:183-195.
local tuple = require "mapreduce.tuple"
-- IEEE-754 binary64 <-> two 32-bit words (big end first) with math.frexp / math.ldexp: Lua 5.2 has no
-- string.pack.  Mirrored 1:1 (and checked against struct.pack) in tests/test_lua_sources.py.
local function double_to_words(x)
  if x == 0 then return 0, 0 end
  local sign = 0
  if x < 0 then sign, x = 0x80000000, -x end
  if x == math.huge then return sign + 0x7FF00000, 0 end
  local m, e = math.frexp(x) -- x = m * 2^e, 0.5 <= m < 1
  e = e + 1022               -- biased exponent of the 1.f form
  local mant
  if e <= 0 then             -- subnormal: 0.f * 2^-1022
    mant, e = m * 2 ^ (52 + e), 0
  else
    mant = (m * 2 - 1) * 2 ^ 52
  end
  local hi_m = math.floor(mant / 2 ^ 32)
  return sign + e * 2 ^ 20 + hi_m, mant - hi_m * 2 ^ 32
end
local function words_to_double(hi, lo)
  local neg = hi >= 0x80000000
  if neg then hi = hi - 0x80000000 end
  local e = math.floor(hi / 2 ^ 20)
  local mant = (hi - e * 2 ^ 20) * 2 ^ 32 + lo
  local x
  if e == 0 then
    x = math.ldexp(mant, -1074)
  elseif e == 2047 then
    x = math.huge -- (NaN is rejected by enc_num, so only infinities arrive here)
  else
    x = math.ldexp(mant + 2 ^ 52, e - 1075)
  end
  return neg and -x or x
end

local function enc_num(x, out, value)
  assert(x == x, value and "NaN cannot be a value" or "NaN cannot be a key")
  local hi, lo
  if value and x == 0 and 1 / x < 0 then
    hi, lo = 0x80000000, 0 -- a value keeps -0
  else
    if x == 0 then x = 0 end -- -0 and 0 are the same table key
    hi, lo = double_to_words(x)
  end
  if hi >= 0x80000000 then hi, lo = 0xFFFFFFFF - hi, 0xFFFFFFFF - lo else hi = hi + 0x80000000 end
  -- 64 bits -> groups of 1,7,7,...,7 bits
  local bits = {}
  for i = 31, 0, -1 do bits[#bits + 1] = math.floor(hi / 2 ^ i) % 2 end
  for i = 31, 0, -1 do bits[#bits + 1] = math.floor(lo / 2 ^ i) % 2 end
  out[#out + 1] = "\16"
  out[#out + 1] = string.char(128 + bits[1])
  for g = 0, 8 do
    local v = 0
    for b = 1, 7 do v = v * 2 + bits[1 + g * 7 + b] end
    out[#out + 1] = string.char(128 + v)
  end
end

local enc_key
local function enc_component(v, out)
  local mt = type(v) == "table" and getmetatable(v)
  if mt == "is_tuple" then
    out[#out + 1] = "\48"
    enc_key(v, out)
  elseif type(v) == "string" then
    assert(not v:find("[%z\1]"), "string components must not contain the bytes 0x00 / 0x01")
    out[#out + 1] = "\32" .. v .. "\1"
  else
    enc_num(assert(tonumber(v), "keys are numbers, strings or tuples of them"), out)
  end
end
enc_key = function(k, out)
  if type(k) == "table" then
    assert(#k <= 31, "tuples of more than 31 components are not supported")
    out[#out + 1] = string.char(128 + #k)
    for i = 1, #k do enc_component(k[i], out) end
  else
    out[#out + 1] = "\127"
    enc_component(k, out)
  end
end

function hbm.encode_key(k)
  local out = {}
  enc_key(tuple(k), out)
  local s = table.concat(out)
  assert(#s <= 123, "encoded key is longer than 123 bytes")
  return s
end

local dec_key
local function dec_component(s, i)
  local tag = s:byte(i)
  if tag == 16 then
    local hi, lo, nb = 0, 0, 0
    for k = 1, 10 do
      local g, w = s:byte(i + k) % 128, (k == 1) and 1 or 7
      for b = w - 1, 0, -1 do
        local bit = math.floor(g / 2 ^ b) % 2
        if nb < 32 then hi = hi * 2 + bit else lo = lo * 2 + bit end
        nb = nb + 1
      end
    end
    if hi >= 0x80000000 then hi = hi - 0x80000000 else hi, lo = 0xFFFFFFFF - hi, 0xFFFFFFFF - lo end
    return words_to_double(hi, lo), i + 11
  elseif tag == 32 then
    local j = s:find("\1", i + 1, true)
    return s:sub(i + 1, j - 1), j + 1
  elseif tag == 48 then
    return dec_key(s, i + 1)
  end
  error("bad component tag")
end
dec_key = function(s, i)
  local head = s:byte(i)
  if head == 127 then return dec_component(s, i + 1) end
  local t, n = {}, head - 128
  i = i + 1
  for k = 1, n do t[k], i = dec_component(s, i) end
  t.n = n
  return tuple(t), i
end
function hbm.decode_key(s) return (dec_key(s, 1)) end

-- Values of value_kind = "bytes" (same format as encode_value / decode_value in ../../mapreduce/tuple.py):
--   value := "\16" num10 (as above, but -0 stays -0) | "\32" bytes (a Lua string: any bytes, any length)
function hbm.encode_value(v)
  if type(v) == "string" then return "\32" .. v end
  assert(type(v) == "number", "values are strings or numbers")
  local out = {}
  enc_num(v, out, true)
  return table.concat(out)
end
function hbm.decode_value(s)
  local tag = s:byte(1)
  if tag == 32 then return s:sub(2) end
  assert(tag == 16 and #s == 11, "bad value encoding")
  return (dec_component(s, 1))
end

-- job_prepare_map (job.lua:154-228): returns the emit closure and the finisher
function hbm.map_job(map_key)
  local m = assert(ctx:map_begin(tostring(map_key)))
  local emit = function(key, value)
    if tuple_keys then key = hbm.encode_key(key) end
    if byte_values then value = hbm.encode_value(value) end
    assert(m:emit(key, value))
  end
  local finish = function(ok)
    if ok then assert(m:commit()) else m:abort() end -- BROKEN jobs publish nothing
  end
  -- a mapfn module declaring hbm_mapfn = "words_file" (value_kind = "bytes"): the device tokenises the file's bytes
  -- and pairs every word with the job value, the file name -- emit(word, value) per token, as an inverted index does
  local words = function(text, value)
    assert(byte_values, "hbm_mapfn = 'words_file' needs value_kind = 'bytes'")
    return assert(m:words_value(text, hbm.encode_value(value)))
  end
  -- a mapfn module declaring hbm_mapfn = "key_numbers_file" (value_kind = "bytes", string keys): the device parses the
  -- file's lines "key number" -- emit(key, tonumber(number)) per line, decimal numbers only
  local key_numbers = function(text)
    assert(byte_values, "hbm_mapfn = 'key_numbers_file' needs value_kind = 'bytes'")
    assert(not tuple_keys, "hbm_mapfn = 'key_numbers_file' needs string keys")
    return assert(m:key_numbers(text))
  end
  return emit, finish, words, key_numbers
end

-- server_prepare_reduce (server.lua:279-329)
function hbm.prepare_reduce()
  if sample_splitters then assert(ctx:sample_splitters()) end
  assert(ctx:shuffle())
  return assert(ctx:partitions())
end

-- job_prepare_reduce (job.lua:230-296): for k,v in hbm.groups(part_key) do ... end
function hbm.groups(part_key)
  local it = assert(ctx:groups(part_key))
  if not tuple_keys and not byte_values then return it end
  return function()
    local k, v = it()
    if k == nil then return nil end
    if byte_values then
      for i = 1, #v do v[i] = hbm.decode_value(v[i]) end
    end
    if tuple_keys then k = hbm.decode_key(k) end
    return k, v
  end
end

function hbm.reset() assert(ctx:reset()) end

return hbm
