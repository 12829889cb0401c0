--[[ modules_b200.lua — nn.Module classes with the reference's names whose updateOutput calls the C ABI.
Loaded INSTEAD of modules/{Foveal,ContextRegion,BBoxNorm}.lua when mpn_backend=b200 (fbcoco.lua:17-21
requires them by name, torch.load finds classes by name), so serialized models keep loading.
No C handle is ever stored in a module field (models are torch.save'd, train.lua:195). UNTESTED here. ]]
local ffi = require 'ffi'
local mpn = paths.dofile('mpn_ffi.lua')
local C = mpn.C

-- nn.Foveal (modules/Foveal.lua) ---------------------------------------------------------------
local Foveal, parent = torch.class('nn.Foveal', 'nn.Module')
function Foveal:__init() parent.__init(self) end
function Foveal:updateOutput(input)
   assert(input:nDimension() == 2)
   assert(input:size(2) == 5)
   if torch.type(input) == 'torch.CudaTensor' then            -- stays on the device (the reference copies to the host and back)
      local cin = input:contiguous()
      self.output:resize(cin:size(1) * 4, 5)
      local ctx = mpn.ctx()
      mpn.check(ctx, C.mpn_foveal_dev(ctx, mpn.fptr(cin), cin:size(1), mpn.fptr(self.output)), 'mpn_foveal_dev')
      return self.output
   end
   local cin = input:float():contiguous()
   local cout = torch.FloatTensor(input:size(1) * 4, 5)
   local ctx = mpn.ctx()
   mpn.check(ctx, C.mpn_foveal(ctx, mpn.fptr(cin), cin:size(1), mpn.fptr(cout)), 'mpn_foveal')
   self.output:resize(cout:size()):copy(cout)
   return self.output
end

-- nn.ContextRegion (modules/ContextRegion.lua) ---------------------------------------------------
local Context, cparent = torch.class('nn.ContextRegion', 'nn.Module')
function Context:__init(scale) cparent.__init(self); self.scale = scale end
function Context:updateOutput(input)
   assert(input:nDimension() == 2)
   assert(input:size(2) == 5)
   if torch.type(input) == 'torch.CudaTensor' then
      local cin = input:contiguous()
      self.output:resize(cin:size())
      local ctx = mpn.ctx()
      mpn.check(ctx, C.mpn_context_region_dev(ctx, mpn.fptr(cin), cin:size(1), self.scale, mpn.fptr(self.output)), 'mpn_context_region_dev')
      return self.output
   end
   local cin = input:float():contiguous()
   local cout = torch.FloatTensor(cin:size())
   local ctx = mpn.ctx()
   mpn.check(ctx, C.mpn_context_region(ctx, mpn.fptr(cin), cin:size(1), self.scale, mpn.fptr(cout)), 'mpn_context_region')
   self.output:resize(cout:size()):copy(cout)
   return self.output
end
function Context:updateGradInput(input, gradOutput)
   self.gradInput:resizeAs(input):zero()
   return self.gradInput
end

-- nn.BBoxNorm (modules/BBoxNorm.lua) -------------------------------------------------------------
local BBoxNorm, bparent = torch.class('nn.BBoxNorm', 'nn.Module')
function BBoxNorm:__init(mean, std)
   assert(mean and std)
   bparent.__init(self)
   self.mean = mean; self.std = std
end
function BBoxNorm:updateOutput(input)
   assert(input:dim() == 2 and input:size(2) % 4 == 0)
   self.output:set(input)
   if not self.train and torch.type(input) == 'torch.CudaTensor' then
      -- evaluate mode on the device: out = in .* std + mean per group of 4 (BBoxNorm.lua:24-29), no host round trip
      self._output = self._output or input.new()
      self._output:resize(input:size()):copy(input)
      local m, s = self.mean:float():contiguous(), self.std:float():contiguous()
      local ctx = mpn.ctx()
      mpn.check(ctx, C.mpn_bbox_norm_dev(ctx, mpn.fptr(self._output), input:size(1), input:size(2), mpn.fptr(m), mpn.fptr(s)), 'mpn_bbox_norm_dev')
      self.output = self._output
   elseif not self.train then
      local x = input:float():contiguous()
      local m, s = self.mean:float():contiguous(), self.std:float():contiguous()
      local ctx = mpn.ctx()
      mpn.check(ctx, C.mpn_bbox_norm(ctx, mpn.fptr(x), x:size(1), x:size(2), mpn.fptr(m), mpn.fptr(s)), 'mpn_bbox_norm')
      self._output = self._output or input.new()
      self._output:resize(x:size()):copy(x)
      self.output = self._output
   end
   return self.output
end
function BBoxNorm:updateGradInput(input, gradOutput)
   assert(self.train, 'cannot updateGradInput in evaluate mode')
   self.gradInput = gradOutput
   return self.gradInput
end
function BBoxNorm:clearState()
   nn.utils.clear(self, '_output')
   return bparent.clearState(self)
end

-- inn.ROIPooling (imagine-nn; vgg.lua:28, model_utils.lua:215) ------------------------------------
-- forward{data, rois}: data N x C x H x W, rois R x 5 [batch idx (1-based), x1, y1, x2, y2] -> R x C x H x W pooled,
-- self.indices = argmax (flat index into the H x W map, -1 for an empty bin). Registered under the same class name so
-- that saved models load.
if not inn then inn = {} end
local ROIPooling, rparent = torch.class('inn.ROIPooling', 'nn.Module')
function ROIPooling:__init(W, H, spatial_scale)
   rparent.__init(self)
   assert(W and H, 'W and H have to be provided')
   self.W, self.H = W, H
   self.spatial_scale = spatial_scale or 1
   self.v2 = true                                           -- post-PR-17 end convention (README.md:202-203)
   self.indices = torch.IntTensor()
end
function ROIPooling:setSpatialScale(scale) self.spatial_scale = scale; return self end
function ROIPooling:updateOutput(input)
   assert(#input == 2)
   local data, rois = input[1], input[2]
   assert(data:nDimension() == 4 and rois:nDimension() == 2 and rois:size(2) == 5)
   local R, nC = rois:size(1), data:size(2)
   local ctx = mpn.ctx()
   if torch.type(data) == 'torch.CudaTensor' then
      -- CudaTensors (the reference's inference path): device pointers straight into mpn_roi_pool_dev, stream-ordered on the
      -- ctx's (= cutorch's default) stream: no host round trip (the reference's Foveal.lua:21-22,42 pattern is NOT reproduced)
      local d, r = data:contiguous(), rois:contiguous()
      self.output = self.output:typeAs(data):resize(R, nC, self.H, self.W)
      self._indices_cuda = self._indices_cuda or torch.CudaIntTensor()
      self._indices_cuda:resize(R, nC, self.H, self.W)
      mpn.check(ctx, C.mpn_roi_pool_dev(ctx, mpn.fptr(d), d:size(1), nC, d:size(3), d:size(4), mpn.fptr(r), R, self.W, self.H,
                                        self.spatial_scale, self.v2 and 2 or 1, mpn.fptr(self.output),
                                        ffi.cast('int32_t*', self._indices_cuda:data())), 'mpn_roi_pool_dev')
      self.indices = self._indices_cuda
      return self.output
   end
   local out = torch.FloatTensor(R, nC, self.H, self.W)
   self.indices = torch.IntTensor(R, nC, self.H, self.W)
   local d, r = data:float():contiguous(), rois:float():contiguous()
   mpn.check(ctx, C.mpn_roi_pool(ctx, mpn.fptr(d), d:size(1), nC, d:size(3), d:size(4), mpn.fptr(r), R, self.W, self.H,
                                 self.spatial_scale, self.v2 and 2 or 1, mpn.fptr(out), ffi.cast('int32_t*', self.indices:data())),
             'mpn_roi_pool')
   self.output = self.output:typeAs(data):resize(out:size()):copy(out)
   return self.output
end
-- backward{data, rois}: gradInput = {grad_data N x C x H x W, zeros R x 5} from the argmax of the last forward. grad_data
-- is summed per cell in ascending (roi, ph, pw) order, so it is deterministic; imagine-nn's backward accumulates with
-- atomics and agrees up to the rounding of that sum. model:backward reaches this module even under nn.NoBackprop trunks
-- (utils.testModel, demo.lua:41), since the towers sit above it.
function ROIPooling:updateGradInput(input, gradOutput)
   assert(#input == 2)
   local data, rois = input[1], input[2]
   local R, N, nC, H, W = rois:size(1), data:size(1), data:size(2), data:size(3), data:size(4)
   local nOut = R * nC * self.H * self.W
   assert(gradOutput:nElement() == nOut, 'gradOutput must be R x C x H x W')
   local ctx = mpn.ctx()
   local gradData
   if torch.type(data) == 'torch.CudaTensor' then
      -- device pointers straight into the _dev entry point, with the forward's device argmax: no host round trip
      assert(self._indices_cuda and self._indices_cuda:nElement() == nOut, 'inn.ROIPooling: updateGradInput needs a forward first')
      local g, r = gradOutput:contiguous(), rois:contiguous()
      self._gradData = self._gradData or data.new()
      self._gradData:resize(N, nC, H, W)
      mpn.check(ctx, C.mpn_roi_pool_backward_dev(ctx, mpn.fptr(g), ffi.cast('int32_t*', self._indices_cuda:data()), N, nC, H, W,
                                                 mpn.fptr(r), R, self.W, self.H, self.spatial_scale, self.v2 and 2 or 1,
                                                 mpn.fptr(self._gradData)), 'mpn_roi_pool_backward_dev')
      gradData = self._gradData
   else
      assert(self.indices:nElement() == nOut, 'inn.ROIPooling: updateGradInput needs a forward first')
      local g, r = gradOutput:float():contiguous(), rois:float():contiguous()
      gradData = torch.FloatTensor(N, nC, H, W)
      mpn.check(ctx, C.mpn_roi_pool_backward(ctx, mpn.fptr(g), ffi.cast('int32_t*', self.indices:data()), N, nC, H, W,
                                             mpn.fptr(r), R, self.W, self.H, self.spatial_scale, self.v2 and 2 or 1,
                                             mpn.fptr(gradData)), 'mpn_roi_pool_backward')
   end
   self._gradRois = self._gradRois or rois.new()
   self._gradRois:resizeAs(rois):zero()
   self.gradInput = {gradData:typeAs(data), self._gradRois}
   return self.gradInput
end
function ROIPooling:clearState()
   self.indices = torch.IntTensor()
   self._indices_cuda = nil
   self._gradData = nil
   self._gradRois = nil
   return rparent.clearState(self)
end
