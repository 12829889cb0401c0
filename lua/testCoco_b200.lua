--[[ testCoco_b200.lua — drop-in for the Coco class of testCoco/coco.lua: the COCOeval score on the device (mpn_coco_eval)
instead of pycocotools through fb.python.

   local Coco = os.getenv('mpn_backend') == 'b200' and paths.dofile('lua/testCoco_b200.lua') or require 'testCoco.coco'

   Coco(annFile)       reads the annotation json with cjson (run_test.lua:10 already requires it)
   Coco:evaluate(boxt) boxt = the N x 7 FloatTensor testCoco/init.lua:65-86 builds; prints COCOeval.summarize's 12 lines and
                       returns the stats as a torch.DoubleTensor(12)

Annotation id 0 is refused (COCO ids start at 1; pycocotools would count a match to it as no match). UNTESTED here (no
LuaJIT); the same entry point is exercised from Python (multipathnet_b200/coco_eval.py, tests/test_coco_eval_gpu.py). ]]
local ffi = require 'ffi'
local cjson = require 'cjson'
local class = require 'class'
local mpn = paths.dofile('mpn_ffi.lua')
local C = mpn.C

local Coco = class('coco')

local function sorted_ids(list)
   local ids, seen = {}, {}
   for _, v in ipairs(list) do
      local id = v.id
      assert(not seen[id], 'duplicate id ' .. tostring(id) .. ' in the annotation file')
      seen[id] = true
      ids[#ids + 1] = id
   end
   table.sort(ids)
   local index = {}
   for i, id in ipairs(ids) do index[id] = i - 1 end
   return ids, index
end

function Coco:__init(annFile)
   local f = assert(io.open(annFile, 'r'), 'cannot open ' .. annFile)
   local d = cjson.decode(f:read('*a')); f:close()
   local img_ids, img_index = sorted_ids(d.images)
   local cat_ids, cat_index = sorted_ids(d.categories)
   local anns = d.annotations or {}
   local G = #anns
   self.n_images, self.n_cats, self.G = #img_ids, #cat_ids, G
   self.image_ids = ffi.new('int64_t[?]', #img_ids)
   for i, id in ipairs(img_ids) do self.image_ids[i - 1] = id end
   self.cat_ids = ffi.new('int64_t[?]', #cat_ids)
   for i, id in ipairs(cat_ids) do self.cat_ids[i - 1] = id end
   local n = math.max(G, 1)
   self.gt_img = ffi.new('int32_t[?]', n); self.gt_cat = ffi.new('int32_t[?]', n); self.gt_crowd = ffi.new('int32_t[?]', n)
   self.gt_box = ffi.new('double[?]', 4 * n); self.gt_area = ffi.new('double[?]', n)
   local ann_seen = {}
   for j, a in ipairs(anns) do
      assert(a.id ~= 0, 'annotation id 0: COCO annotation ids start at 1')
      assert(not ann_seen[a.id], 'duplicate annotation id ' .. tostring(a.id)); ann_seen[a.id] = true
      local ii, ci = img_index[a.image_id], cat_index[a.category_id]
      assert(ii and ci, 'annotation ' .. tostring(a.id) .. ' refers to an unknown image or category')
      self.gt_img[j - 1], self.gt_cat[j - 1] = ii, ci
      self.gt_crowd[j - 1] = a.iscrowd or 0
      for c = 1, 4 do self.gt_box[4 * (j - 1) + c - 1] = a.bbox[c] end
      self.gt_area[j - 1] = a.area
   end
end

local TITLES = {
   {1, '0.50:0.95', 'all', 100}, {1, '0.50', 'all', 100}, {1, '0.75', 'all', 100}, {1, '0.50:0.95', 'small', 100},
   {1, '0.50:0.95', 'medium', 100}, {1, '0.50:0.95', 'large', 100}, {0, '0.50:0.95', 'all', 1}, {0, '0.50:0.95', 'all', 10},
   {0, '0.50:0.95', 'all', 100}, {0, '0.50:0.95', 'small', 100}, {0, '0.50:0.95', 'medium', 100}, {0, '0.50:0.95', 'large', 100},
}

function Coco:evaluate(res)
   local rows = res:float():contiguous()
   local D = rows:nElement() > 0 and rows:size(1) or 0
   local K = self.n_cats
   local precision = torch.DoubleTensor(10, 101, K, 4, 3)
   local recall = torch.DoubleTensor(10, K, 4, 3)
   local stats = torch.DoubleTensor(12)
   local ctx = mpn.ctx()
   mpn.check(ctx, C.mpn_coco_eval(ctx, self.n_images, self.image_ids, K, self.cat_ids, self.G, self.gt_img, self.gt_cat,
                                  self.gt_box, self.gt_area, self.gt_crowd, D, mpn.fptr(rows),
                                  ffi.cast('double*', precision:data()), ffi.cast('double*', recall:data()),
                                  ffi.cast('double*', stats:data())), 'mpn_coco_eval')
   for i, t in ipairs(TITLES) do
      local title, kind = t[1] == 1 and 'Average Precision' or 'Average Recall', t[1] == 1 and '(AP)' or '(AR)'
      print(string.format(' %-18s %s @[ IoU=%-9s | area=%6s | maxDets=%3d ] = %0.3f', title, kind, t[2], t[3], t[4], stats[i]))
   end
   self.precision, self.recall = precision, recall
   return stats
end

return Coco
