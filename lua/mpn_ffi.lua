--[[ mpn_ffi.lua — LuaJIT-FFI binding of libmpn_b200.so (include/mpn_abi.h).

Same mechanism the reference already uses for its only native code (utils.lua:15-26:
ffi.cdef + ffi.load of ./libnms.so). The cdef text is the block between MPN_CDEF_BEGIN and
MPN_CDEF_END of include/mpn_abi.h, read at load time so there is one source of truth.

UNTESTED IN THE BUILD ENVIRONMENT: Torch-7 / LuaJIT are not installed there (SURVEY top table);
the same C ABI is exercised from Python (multipathnet_b200/_lib.py, tests/). ]]
local ffi = require 'ffi'

local M = {}

local function read_cdef(path)
   local f = assert(io.open(path, 'r'), 'cannot open ' .. path)
   local src = f:read('*a'); f:close()
   local body = src:match('MPN_CDEF_BEGIN %*/(.-)/%* MPN_CDEF_END')
   assert(body, 'MPN_CDEF markers not found in ' .. path)
   return body
end

local here = debug.getinfo(1, 'S').source:match('^@(.*)/[^/]*$') or '.'
ffi.cdef(read_cdef(here .. '/../include/mpn_abi.h'))

local ok, C = pcall(ffi.load, here .. '/../multipathnet_b200/libmpn_b200.so')
if not ok then
   os.execute('make -C ' .. here .. '/..')          -- same auto-build convention as utils.lua:21-26
   ok, C = pcall(ffi.load, here .. '/../multipathnet_b200/libmpn_b200.so')
   assert(ok, 'run make and check what is wrong (libmpn_b200.so needs nvcc with sm_90a)')
end
M.C = C

-- one context per (Lua state, device): test_runner.lua:55-66 runs one Lua state per GPU thread
local ctxs = {}
function M.ctx()
   local dev = cutorch and (cutorch.getDevice() - 1) or 0
   if not ctxs[dev] then
      local out = ffi.new('mpn_ctx*[1]')
      -- default: nil stream = the legacy default stream (cutorch's default), so ordering with surrounding Torch ops is kept.
      -- mpn_replica_streams=1: a stream of its own, for several donkey threads (model replicas) per GPU whose kernels should
      -- overlap (INTEGRATION.md section 5); CudaTensors handed to _dev entry points must then be synchronised by the caller.
      local rc
      if os.getenv('mpn_replica_streams') == '1' then rc = C.mpn_ctx_create_stream(dev, 0, out)
      else rc = C.mpn_ctx_create(dev, nil, out) end
      if rc ~= 0 then error('mpn_ctx_create: ' .. ffi.string(C.mpn_last_error(nil))) end
      ctxs[dev] = ffi.gc(out[0], C.mpn_ctx_destroy)
   end
   return ctxs[dev]
end

function M.check(ctx, rc, what)
   if rc ~= 0 then error((what or 'mpn') .. ': ' .. ffi.string(C.mpn_last_error(ctx))) end
end

-- raw float* of a contiguous Float/Cuda tensor (tensor:data() is the FFI pointer in torch7/cutorch)
function M.fptr(t)
   assert(t:isContiguous(), 'tensor must be contiguous')
   return ffi.cast('float*', t:data())
end

return M
