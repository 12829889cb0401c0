--[[ model_desc.lua — nn graph -> mpn_model_desc -> mpn_model_create (include/mpn_abi.h).

Walks the nn.Sequential a model file returns (models/vgg.lua:23-31, models/resnet.lua:28-50,
models/multipathnet.lua:30-121) and describes it as data for libmpn_b200.so: the trunk and every per-ROI tower as lists
of conv / pool / flatten layers on numbered slots, the towers' pooled trunk taps, the class / bbox heads as column ranges.
It is the Lua twin of multipathnet_b200/t7.py:model_from_t7 (same table algebra, same folds), which the CPU suite
checks against a module-by-module evaluation of hand-assembled graphs (tests/test_t7_graphs_cpu.py):
  * containers (Sequential, NoBackprop, DataParallelTable, ConcatTable, ParallelTable, FlattenTable, SelectTable) are
    evaluated symbolically: a value is a slot number or a table of values;
  * ConcatTable{branch, shortcut} + CAddTable + ReLU becomes a convolution with a residual input (fb.resnet.torch);
  * nn.Concat(2) / nn.DepthConcat(2) (inceptionv3.lua's Mixed blocks, nested): the layers that end each branch write
    their channel slices of one slot; they, 1 x n / n x 1 convolutions with a pad per axis and windowed average pools
    (count_include_pad, ceil_mode) go to the library as mpn_layer_ext records through mpn_model_create_ext;
  * SpatialBatchNormalization / inn.ConstAffine / MulConstant directly after a convolution are folded into it
    (inn.utils.foldBatchNorm, resnet.lua:33-36); conv345Combine's per-level MulConstant factors are folded into conv_mix.
Weights are handed over as host FloatTensors and copied by mpn_model_create; nothing here stays referenced by the
library. The returned table {handle, num_classes} is what lua/ImageDetect_b200.lua takes as `model`; the handle is
freed by ffi.gc and must not be stored in a serialisable field (models are torch.save'd, train.lua:195).

UNTESTED IN THE BUILD ENVIRONMENT (no Torch-7 / LuaJIT there). ]]
local ffi = require 'ffi'
local mpn = paths.dofile('mpn_ffi.lua')
local C = mpn.C

local CONV, MAXPOOL, AVGPOOL, FLATTEN, AVGPOOL_WIN = 1, 2, 3, 4, 6   -- MPN_LAYER_* (mpn_abi.h)
local LRN = 5                                                         -- MPN_LAYER_LRN: CaffeNet's norm1 / norm2
-- the cross-map LRN modules (nn, cudnn: SpatialCrossMapLRN; inn: SpatialCrossResponseNormalization)
local LRN_MODULES = {SpatialCrossMapLRN = true, SpatialCrossResponseNormalization = true}
local PASS = {Identity = true, Copy = true, Contiguous = true, View = true, Reshape = true, Transpose = true, Squeeze = true}

local function base(m) return (torch.type(m):gsub('^[^.]*%.', '')) end
local function f32(t) return t:float():contiguous() end

-- ---------------------------------------------------------------------------------------------- layer list builder
local Layers = {}
Layers.__index = Layers

local function new_layers(cin, h, w)
   return setmetatable({layers = {}, next = 1, shape = {[0] = {cin, h, w}}}, Layers)
end

function Layers:slot(c, h, w)
   local s = self.next
   self.next = s + 1
   self.shape[s] = {c, h, w}
   return s
end

function Layers:producer(slot)
   for i = #self.layers, 1, -1 do
      if self.layers[i].out_slot == slot then return self.layers[i], i end
   end
end

function Layers:open_conv(slot, what)
   local L = self:producer(slot)
   assert(L and L.kind == CONV and L.relu == 0 and L.residual_slot < 0 and (L.out_c_total or 0) == 0,
          what .. ' that does not directly follow a convolution / Linear')
   return L
end

-- y = scale[c] * x + shift[c] right after a convolution: fold into its weight and bias
function Layers:affine(slot, scale, shift, what)
   local L = self:open_conv(slot, what)
   assert(scale:nElement() == L.cout and shift:nElement() == L.cout, what .. ': channel count mismatch')
   local w = L.w:double()
   local s = scale:double():view(L.cout, 1):expand(L.cout, w:nElement() / L.cout)
   L.w = w:view(L.cout, -1):cmul(s):float():viewAs(L.w):contiguous()
   L.b = L.b:double():cmul(scale:double()):add(shift:double()):float()
end

local function pool_out(n, k, s, p, ceil)                  -- nn.SpatialMaxPooling output size
   local o
   if ceil then o = math.ceil((n + 2 * p - k) / s) + 1 else o = math.floor((n + 2 * p - k) / s) + 1 end
   if ceil and (o - 1) * s >= n + p then o = o - 1 end
   return o
end

-- nn.Concat(2) / nn.DepthConcat(2): every branch runs on v; the layers that write each branch's output are re-targeted to
-- their channel slice of one slot (out_c_off / out_c_total), nested concatenations included
function Layers:concat(m, b, v)
   assert(type(v) == 'number', 'nn.' .. b .. ' applied to a table')
   assert((m.dimension or 2) == 2, 'nn.' .. b .. ' along dimension ' .. tostring(m.dimension) .. ': only the channel dimension (2) is concatenated')
   local outs, total = {}, 0
   for _, c in ipairs(m.modules) do
      local first = base(c) == 'Sequential' and c.modules[1] or c
      assert(base(first) ~= 'Narrow', 'nn.' .. b .. " of nn.Narrow branches (loadcaffe's form of a grouped convolution): convert it " ..
             'to cudnn.SpatialConvolution with groups')
   end
   for i, c in ipairs(m.modules) do
      local o = self:run(c, v)
      assert(type(o) == 'number' and o ~= v, 'nn.' .. b .. ' branch that is empty or returns a table')
      local sh, s1 = self.shape[o], self.shape[outs[1] or o]
      assert(sh[2] == s1[2] and sh[3] == s1[3], 'nn.' .. b .. ' of branches with different map sizes')
      outs[i] = o; total = total + sh[1]
   end
   local o = self:slot(total, self.shape[outs[1]][2], self.shape[outs[1]][3])
   local off = 0
   for _, br in ipairs(outs) do
      local n = 0
      for _, L in ipairs(self.layers) do
         assert(L.in_slot ~= br and L.residual_slot ~= br, 'nn.' .. b .. ' branch output read inside the block')
         if L.out_slot == br then
            assert((L.kind == CONV or L.kind == MAXPOOL or L.kind == AVGPOOL_WIN) and L.residual_slot < 0,
                   'nn.' .. b .. ' branch that does not end in a convolution or a pooling')
            L.out_c_off = off + ((L.out_c_total or 0) > 0 and L.out_c_off or 0)
            L.out_c_total, L.out_slot = total, o
            n = n + 1
         end
      end
      assert(n > 0, 'nn.' .. b .. ' branch without a layer')
      off = off + self.shape[br][1]
   end
   return o
end

function Layers:run(m, v)
   local b = base(m)
   if b == 'Sequential' or b == 'NoBackprop' then
      for _, c in ipairs(m.modules) do v = self:run(c, v) end
      return v
   elseif b == 'DataParallelTable' or b == 'DataParallel' then
      return self:run(m.modules[1], v)
   elseif b == 'ConcatTable' then
      local out = {}
      for i, c in ipairs(m.modules) do out[i] = self:run(c, v) end
      return out
   elseif b == 'ParallelTable' then
      assert(type(v) == 'table' and #v == #m.modules, 'nn.ParallelTable arity does not match its input table')
      local out = {}
      for i, c in ipairs(m.modules) do out[i] = self:run(c, v[i]) end
      return out
   elseif b == 'Concat' or b == 'DepthConcat' then
      return self:concat(m, b, v)
   elseif b == 'FlattenTable' then
      local out = {}
      local function flat(x)
         if type(x) == 'table' then for _, e in ipairs(x) do flat(e) end else out[#out + 1] = x end
      end
      flat(v)
      return out
   elseif b == 'SelectTable' then
      assert(type(v) == 'table', 'nn.SelectTable on a tensor')
      return m.index > 0 and v[m.index] or v[#v + m.index + 1]
   elseif PASS[b] then
      return v
   elseif b == 'Dropout' then
      assert(m.v2 ~= false, 'nn.Dropout(v2=false) scales at test time')
      return v
   elseif b == 'CAddTable' then
      assert(type(v) == 'table' and #v == 2 and type(v[1]) == 'number' and type(v[2]) == 'number',
             'nn.CAddTable of anything but two tensors')
      for _, pair in ipairs{{v[1], v[2]}, {v[2], v[1]}} do
         local main, other = pair[1], pair[2]
         local L, idx = self:producer(main)
         local sa, sb = self.shape[main], self.shape[other]
         if L and L.kind == CONV and L.relu == 0 and L.residual_slot < 0
            and sa[1] == sb[1] and sa[2] == sb[2] and sa[3] == sb[3] then
            table.remove(self.layers, idx)                 -- the shortcut branch was emitted after it: run it last
            table.insert(self.layers, L)
            L.residual_slot = other
            return main
         end
      end
      error('residual add whose branches do not end in a bare convolution')
   end
   assert(type(v) == 'number', torch.type(m) .. ' applied to a table')
   local s = v
   local c, h, w = self.shape[s][1], self.shape[s][2], self.shape[s][3]
   if b == 'SpatialConvolution' or b == 'SpatialConvolutionMM' then
      local g = m.groups or 1                              -- a grouped convolution (CaffeNet's conv2 / 4 / 5): a groups record
      assert(g >= 1 and m.nInputPlane % g == 0 and m.nOutputPlane % g == 0 and (m.nInputPlane / g) % 8 == 0 and
             (m.nOutputPlane / g) % 8 == 0, 'grouped convolution: each group must read and write a multiple of 8 channels')
      local pad_w, pad = m.padW or 0, m.padH or m.padW or 0   -- a pad per axis: 1 x n / n x 1 kernels (inceptionv3.lua)
      assert(m.dW == m.dH, 'anisotropic stride: the engine strides both axes alike')
      assert(m.nInputPlane == c, 'conv input planes do not match its input')
      local o = self:slot(m.nOutputPlane, h and math.floor((h + 2 * pad - m.kH) / m.dH) + 1,
                          w and math.floor((w + 2 * pad_w - m.kW) / m.dW) + 1)
      table.insert(self.layers, {kind = CONV, in_slot = s, out_slot = o, cin = c, cout = m.nOutputPlane, kh = m.kH, kw = m.kW,
                                 stride = m.dW, pad = pad, pad_w = pad_w, relu = 0, residual_slot = -1, ceil_mode = 0, groups = g,
                                 w = f32(m.weight):view(m.nOutputPlane, c / g, m.kH, m.kW),
                                 b = m.bias and f32(m.bias) or torch.FloatTensor(m.nOutputPlane):zero()})
      return o
   elseif b == 'Linear' or b == 'LinearNB' then
      if h and h * w > 1 then                              -- View(-1):setNumInputDims(3) before the first Linear
         local s2 = self:slot(c * h * w, 1, 1)
         table.insert(self.layers, {kind = FLATTEN, in_slot = s, out_slot = s2, cin = 0, cout = 0, kh = 1, kw = 1, stride = 1,
                                    pad = 0, relu = 0, residual_slot = -1, ceil_mode = 0})
         s, c = s2, c * h * w
      end
      local nout = m.weight:size(1)
      assert(m.weight:size(2) == c, 'Linear input size does not match its input')
      local o = self:slot(nout, 1, 1)
      -- nn.LinearNB, the biasless first factor utils.SVDlinear leaves behind, gets no bias (index -1, as svd_compress)
      local bias = nil
      if b == 'Linear' then bias = m.bias and f32(m.bias) or torch.FloatTensor(nout):zero() end
      table.insert(self.layers, {kind = CONV, in_slot = s, out_slot = o, cin = c, cout = nout, kh = 1, kw = 1, stride = 1, pad = 0,
                                 relu = 0, residual_slot = -1, ceil_mode = 0, w = f32(m.weight), b = bias})
      return o
   elseif b == 'SpatialBatchNormalization' or b == 'BatchNormalization' then
      local inv
      if m.running_var then inv = m.running_var:double():add(m.eps or 1e-5):sqrt():pow(-1)
      elseif m.running_std then inv = m.running_std:double()          -- older nn: already 1 / sqrt(var + eps)
      else error('batch normalisation without running statistics') end
      local scale = m.weight and m.weight:double():cmul(inv) or inv
      local shift = m.running_mean:double():cmul(scale):mul(-1)
      if m.bias then shift:add(m.bias:double()) end
      self:affine(s, scale, shift, torch.type(m))
      return s
   elseif b == 'ConstAffine' then                          -- inn.utils.BNtoFixed: y = a * x + b per channel
      self:affine(s, m.a, m.b, torch.type(m))
      return s
   elseif b == 'MulConstant' then
      self:affine(s, torch.DoubleTensor(c):fill(m.constant_scalar), torch.DoubleTensor(c):zero(), torch.type(m))
      return s
   elseif b == 'ReLU' then
      local L = self:producer(s)
      assert(L and L.kind == CONV and (L.out_c_total or 0) == 0, 'ReLU that does not follow a convolution / Linear / residual add')
      L.relu = 1
      return s
   elseif LRN_MODULES[b] then
      assert(m.size == 5 and m.alpha == 1e-4 and m.beta == 0.75 and (m.k or 1) == 1,
             "only CaffeNet's LRN (size 5, alpha 1e-4, beta 0.75, k 1) runs on the device")
      assert(c % 8 == 0, 'LRN over a number of channels that is not a multiple of 8')
      local o = self:slot(c, h, w)
      table.insert(self.layers, {kind = LRN, in_slot = s, out_slot = o, cin = 0, cout = 0, kh = 1, kw = 1, stride = 1, pad = 0,
                                 relu = 0, residual_slot = -1, ceil_mode = 0})
      return o
   elseif b == 'SpatialMaxPooling' then
      assert(m.kW == m.kH and m.dW == m.dH, 'anisotropic pooling')
      local pad, ceil = m.padW or 0, m.ceil_mode and true or false
      local o = self:slot(c, h and pool_out(h, m.kH, m.dH, pad, ceil), w and pool_out(w, m.kW, m.dW, pad, ceil))
      table.insert(self.layers, {kind = MAXPOOL, in_slot = s, out_slot = o, cin = 0, cout = 0, kh = m.kH, kw = m.kW, stride = m.dW,
                                 pad = pad, relu = 0, residual_slot = -1, ceil_mode = ceil and 1 or 0})
      return o
   elseif b == 'SpatialAveragePooling' then
      local pad = m.padW or 0
      if h and m.kH == h and m.kW == w and pad == 0 then   -- the global pool that ends a ResNet (resnet.lua:39)
         local o = self:slot(c, 1, 1)
         table.insert(self.layers, {kind = AVGPOOL, in_slot = s, out_slot = o, cin = 0, cout = 0, kh = 1, kw = 1, stride = 1, pad = 0,
                                    relu = 0, residual_slot = -1, ceil_mode = 0})
         return o
      end
      assert(m.kW == m.kH and m.dW == m.dH and pad == (m.padH or 0), 'anisotropic average pooling')
      local ceil = m.ceil_mode and true or false
      local o = self:slot(c, h and pool_out(h, m.kH, m.dH, pad, ceil), w and pool_out(w, m.kW, m.dW, pad, ceil))
      table.insert(self.layers, {kind = AVGPOOL_WIN, in_slot = s, out_slot = o, cin = 0, cout = 0, kh = m.kH, kw = m.kW, stride = m.dW,
                                 pad = pad, relu = 0, residual_slot = -1, ceil_mode = ceil and 1 or 0,
                                 exclude_pad = (m.count_include_pad == false) and 1 or 0})   -- setCountExcludePad
      return o
   end
   error('module ' .. torch.type(m) .. ' is not on the accelerated path')
end

-- ---------------------------------------------------------------------------------------------------- graph walk
local function parse_pool_level(seq, trunk_vals)             -- make1PoolingLayer, model_utils.lua:212-228
   local k = seq.modules
   assert(base(k[1]) == 'ParallelTable' and base(k[2]) == 'ROIPooling', 'pooling branch is not {SelectTable, Identity} + inn.ROIPooling')
   local sel = k[1].modules[1]
   assert(base(sel) == 'SelectTable', 'pooling branch does not select a trunk output')
   local level = {slot = trunk_vals[sel.index], W = k[2].W, H = k[2].H, scale = k[2].spatial_scale, norm = false, factor = 1}
   for i = 3, #k do
      local b = base(k[i])
      if b == 'Normalize' then assert(k[i].p == 2, 'nn.Normalize with p ~= 2'); level.norm = true
      elseif b == 'MulConstant' then level.factor = level.factor * k[i].constant_scalar
      else assert(PASS[b], 'pooling branch module ' .. torch.type(k[i])) end
   end
   return level
end

local function heads_of(mods, width, narrows)                -- classAndBBoxLinear (+ integral rewrite), model_utils.lua:105-119,275-317
   assert(#mods == 2, 'expected {class head(s), bbox head}')
   local cols = narrows or {{0, width}, {0, width}}
   local cls_m = base(mods[1]) == 'ConcatTable' and mods[1].modules or {mods[1]}
   local function head(m, col)
      assert(base(m) == 'Linear' and m.weight:size(2) == col[2], 'head Linear does not match its columns')
      return {col_begin = col[1], col_len = col[2], cout = m.weight:size(1), w = f32(m.weight),
              b = m.bias and f32(m.bias) or torch.FloatTensor(m.weight:size(1)):zero()}
   end
   local cls = {}
   for i, m in ipairs(cls_m) do cls[i] = head(m, cols[1]) end
   return cls, head(mods[2], cols[2])
end

local M = {}

-- model: the nn.Sequential detection model; opt: {max_rois = 2048, max_h = 1024, max_w = 1344, roi_variant = 2}
function M.create(model, opt)
   opt = opt or {}
   assert(base(model) == 'Sequential', 'expected the nn.Sequential detection model')
   local top = model.modules
   assert(base(top[1]) == 'ParallelTable' and #top[1].modules == 2, 'expected nn.ParallelTable{trunk, Identity} first (vgg.lua:23-27)')
   local tb = new_layers(3)
   local tv = tb:run(top[1].modules[1], 0)
   local trunk_vals = type(tv) == 'table' and tv or {tv}
   local towers, widths, i = {}, {}, 2

   if base(top[2]) == 'ROIPooling' then
      assert(#trunk_vals == 1, 'inn.ROIPooling on a trunk that returns several maps')
      local roi = top[2]
      local lb = new_layers(tb.shape[trunk_vals[1]][1], roi.H, roi.W)
      local v = 0
      i = 3
      while top[i] and base(top[i]) ~= 'ConcatTable' and base(top[i]) ~= 'ParallelTable' do
         v = lb:run(top[i], v)
         i = i + 1
      end
      local sh = lb.shape[v]
      if sh[2] * sh[3] > 1 then
         local v2 = lb:slot(sh[1] * sh[2] * sh[3], 1, 1)
         table.insert(lb.layers, {kind = FLATTEN, in_slot = v, out_slot = v2, cin = 0, cout = 0, kh = 1, kw = 1, stride = 1, pad = 0,
                                  relu = 0, residual_slot = -1, ceil_mode = 0})
         v = v2
      end
      towers[1] = {region = 0, levels = {{slot = trunk_vals[1], scale = roi.spatial_scale}}, pooled_w = roi.W, pooled_h = roi.H,
                   normalize = 0, layers = lb.layers, out_slot = v}
      widths[1] = lb.shape[v][1]
   else
      assert(base(top[2]) == 'ParallelTable' and base(top[3]) == 'ModelParallelTable',
             'expected inn.ROIPooling or the foveal ModelParallelTable after the trunk')
      assert(top[3].dimension == 2, 'ModelParallelTable joining along a dimension other than 2')
      for _, t in ipairs(top[3].modules) do
         local k = t.modules
         local sel = k[1].modules[2]
         assert(base(sel) == 'Select' and sel.dimension == 1, 'tower does not nn.Select(1, region) its ROIs')
         local levels, post, lb, v = {}, 1, nil, 0
         for _, m in ipairs(k[2].modules) do                -- conv345Combine, model_utils.lua:209-251
            local b = base(m)
            if b == 'ConcatTable' and #levels == 0 then
               for _, br in ipairs(m.modules) do levels[#levels + 1] = parse_pool_level(br, trunk_vals) end
            elseif b == 'JoinTable' then
               assert(m.dimension == 2, 'levels are joined along channels')
            elseif b == 'MulConstant' and not lb then
               post = post * m.constant_scalar
            elseif (b == 'SpatialConvolution' or b == 'SpatialConvolutionMM') and not lb then
               local tot = 0
               for _, l in ipairs(levels) do
                  assert(l.W == levels[1].W and l.H == levels[1].H and l.norm == levels[1].norm, 'levels pooled differently')
                  tot = tot + tb.shape[l.slot][1]
               end
               lb = new_layers(tot, levels[1].H, levels[1].W)
               v = lb:run(m, 0)
               -- the kernel applies Normalize + MulConstant(1000) itself; anything else is folded into conv_mix's input columns
               local L, c0 = lb.layers[1], 0
               local w = L.w:double()
               for _, l in ipairs(levels) do
                  local n = tb.shape[l.slot][1]
                  w:narrow(2, c0 + 1, n):mul(l.factor * (levels[1].norm and post / 1000 or post))
                  c0 = c0 + n
               end
               L.w = w:float()
            else
               assert(PASS[b], 'conv345Combine module ' .. torch.type(m))
            end
         end
         assert(lb, 'tower without conv_mix (model_utils.lua:242)')
         for j = 3, #k do v = lb:run(k[j], v) end
         local lv = {}
         for j, l in ipairs(levels) do lv[j] = {slot = l.slot, scale = l.scale} end
         towers[#towers + 1] = {region = sel.index - 1, levels = lv, pooled_w = levels[1].W, pooled_h = levels[1].H,
                                normalize = levels[1].norm and 1 or 0, layers = lb.layers, out_slot = v}
         widths[#widths + 1] = lb.shape[v][1]
      end
      i = 4
   end

   local total = 0
   for _, wd in ipairs(widths) do total = total + wd end
   local narrows, cls, bbox
   local no_softmax, has_norm = model.noSoftMax and 1 or 0, 0
   local mean, std = {0, 0, 0, 0}, {0.1, 0.1, 0.2, 0.2}
   local function take_norm(n)
      has_norm = 1
      for j = 1, 4 do mean[j] = n.mean:view(-1)[j]; std[j] = n.std:view(-1)[j] end
   end
   while top[i] do
      local m, b = top[i], base(top[i])
      if b == 'ConcatTable' and not cls and base(m.modules[1]) == 'Narrow' then        -- multipathnet.lua:115
         narrows = {}
         for j, n in ipairs(m.modules) do assert(n.dimension == 2); narrows[j] = {n.index - 1, n.length} end
      elseif (b == 'ConcatTable' or b == 'ParallelTable') and not cls then
         cls, bbox = heads_of(m.modules, total, narrows)
      elseif b == 'ModeSwitch' then
         no_softmax = 1                                    -- eval branch = mean of the K softmaxes
      elseif b == 'ParallelTable' then
         for _, n in ipairs(m.modules) do if base(n) == 'BBoxNorm' then take_norm(n) end end
      elseif b == 'BBoxNorm' then
         take_norm(m)
      else
         assert(b == 'SoftMax' or PASS[b], 'head module ' .. torch.type(m))
      end
      i = i + 1
   end
   assert(cls, 'no {class, bbox} head found')
   if #cls > 1 then no_softmax = 1 end

   -- ---- flatten into the C structs; `keep` holds every tensor / cdata alive until mpn_model_create has copied them
   local keep, wts = {}, {}
   local function widx(t)
      if not t then return -1 end
      wts[#wts + 1] = t:contiguous()
      return #wts - 1
   end
   local function fill_layers(list)
      local arr = ffi.new('mpn_layer[?]', math.max(#list, 1))
      for j, L in ipairs(list) do
         local d = arr[j - 1]
         d.kind, d.in_slot, d.out_slot = L.kind, L.in_slot, L.out_slot
         d.cin, d.cout, d.kh, d.kw, d.stride, d.pad = L.cin, L.cout, L.kh, L.kw, L.stride, L.pad
         d.relu, d.residual_slot, d.ceil_mode = L.relu, L.residual_slot, L.ceil_mode
         d.weight, d.bias = widx(L.w), widx(L.b)
      end
      keep[#keep + 1] = arr
      return arr
   end
   local desc = ffi.new('mpn_model_desc')
   desc.n_trunk_layers, desc.trunk_layers = #tb.layers, fill_layers(tb.layers)
   local all_tl = {}
   local tw = ffi.new('mpn_tower[?]', #towers)
   for j, t in ipairs(towers) do
      local d = tw[j - 1]
      d.region, d.n_levels = t.region, #t.levels
      for l, lv in ipairs(t.levels) do d.level_slot[l - 1] = lv.slot; d.level_scale[l - 1] = lv.scale end
      d.pooled_w, d.pooled_h, d.normalize = t.pooled_w, t.pooled_h, t.normalize
      d.n_layers, d.first_layer, d.out_slot = #t.layers, #all_tl, t.out_slot
      for _, L in ipairs(t.layers) do all_tl[#all_tl + 1] = L end
   end
   desc.n_towers, desc.towers = #towers, tw
   desc.n_tower_layers, desc.tower_layers = #all_tl, fill_layers(all_tl)
   local function fill_head(d, h)
      d.col_begin, d.col_len, d.cout, d.weight, d.bias = h.col_begin, h.col_len, h.cout, widx(h.w), widx(h.b)
   end
   local ch = ffi.new('mpn_head[?]', #cls)
   for j, h in ipairs(cls) do fill_head(ch[j - 1], h) end
   desc.n_cls_heads, desc.cls_heads = #cls, ch
   fill_head(desc.bbox_head, bbox)
   desc.num_classes = cls[1].cout
   desc.roi_variant = opt.roi_variant or 2
   desc.no_softmax, desc.has_bbox_norm = no_softmax, has_norm
   for j = 1, 4 do desc.bbox_mean[j - 1] = mean[j]; desc.bbox_std[j - 1] = std[j] end
   desc.max_rois, desc.max_h, desc.max_w = opt.max_rois or 2048, opt.max_h or 1024, opt.max_w or 1344

   local wp = ffi.new('const float*[?]', #wts)
   local ne = ffi.new('int64_t[?]', #wts)
   for j, t in ipairs(wts) do wp[j - 1] = mpn.fptr(t); ne[j - 1] = t:nElement() end
   for _, x in ipairs{desc, tw, ch, wp, ne, wts} do keep[#keep + 1] = x end
   -- mpn_layer_ext records (include/mpn_abi.h) for the layers that need more than mpn_layer says: none for VGG, MultiPathNet,
   -- ResNet and NIN, which keep mpn_model_create
   local ext = {}
   local function add_ext(tower, list)
      for j, L in ipairs(list) do
         local pw = L.pad_w or L.pad
         assert(tower < 0 or ((L.groups or 1) == 1 and L.kind ~= LRN), 'a grouped convolution or an LRN runs in the trunk only')
         if pw ~= L.pad or (L.out_c_total or 0) > 0 or (L.exclude_pad or 0) ~= 0 or (L.groups or 1) > 1 then
            ext[#ext + 1] = {tower, j - 1, pw, L.out_c_off or 0, L.out_c_total or 0, L.exclude_pad or 0, (L.groups or 1) > 1 and L.groups or 0}
         end
      end
   end
   add_ext(-1, tb.layers)
   for j, t in ipairs(towers) do add_ext(j - 1, t.layers) end
   local out = ffi.new('mpn_model*[1]')
   local ctx = mpn.ctx()
   if #ext > 0 then
      local ea = ffi.new('mpn_layer_ext[?]', #ext)
      for j, e in ipairs(ext) do
         local d = ea[j - 1]
         d.tower, d.layer, d.pad_w, d.out_c_off, d.out_c_total, d.exclude_pad, d.groups = e[1], e[2], e[3], e[4], e[5], e[6], e[7]
      end
      keep[#keep + 1] = ea
      mpn.check(ctx, C.mpn_model_create_ext(ctx, desc, ea, #ext, wp, ne, #wts, out), 'mpn_model_create_ext')
   else
      mpn.check(ctx, C.mpn_model_create(ctx, desc, wp, ne, #wts, out), 'mpn_model_create')
   end
   keep = nil                                              -- everything was copied
   return {handle = ffi.gc(out[0], C.mpn_model_destroy), num_classes = desc.num_classes}
end

return M
