// test_offload.cpp -- GPU memory offloading through the C++ adapters (gtsam_points_b200.hpp): the reference's OffloadableGPU calls
// on PointCloudGPU and GaussianVoxelMapGPU through OffloadableGPU::Ptr, and factors with set_enable_offloading(true) driven in the
// optimizers' call order (set.add(f) -> set.calc_linear_factors(values) -> set.error(values) -> f->error(values)) while every object
// they read is offloaded.  Their linearizations and errors must equal, bit for bit, those of the same factors over resident
// objects.  Built standalone and with -I tests/cpp/mock_gtsam by tests/test_offload_cpp.py.
//   usage: test_offload <case.bin>
#include "driver.hpp"

typedef struct CUstream_st* cudaStream_t;  // driver_types.h's own declaration: the stream type reference code passes

// The reference's calls with a stream (IntegratedVGICPDerivatives::touch_points: target_->touch(stream)), through the base class.
// Each of them is an offload, a reload and a touch of a resident object.
static bool with_stream(const OffloadableGPU::Ptr& o, cudaStream_t stream) { return o->offload_gpu(stream) && o->reload_gpu(stream) && !o->touch(stream); }

static bool same_hess(const Hess& a, const Hess& b) {
  return a.binary == b.binary && std::memcmp(a.G11, b.G11, sizeof(a.G11)) == 0 && std::memcmp(a.G12, b.G12, sizeof(a.G12)) == 0 &&
         std::memcmp(a.G22, b.G22, sizeof(a.G22)) == 0 && std::memcmp(a.g1, b.g1, sizeof(a.g1)) == 0 && std::memcmp(a.g2, b.g2, sizeof(a.g2)) == 0 &&
         std::memcmp(&a.f, &b.f, sizeof(a.f)) == 0;
}

// One optimizer step over `factors`: the batched linearization at `values`, then the batched evaluation at `values2`
static void step(const std::vector<std::shared_ptr<IntegratedMatchingCostFactorB200>>& factors, const Values& values, const Values& values2, std::vector<Hess>& lin,
                 std::vector<double>& err) {
  std::shared_ptr<FactorSetBase> set = create_nonlinear_factor_set_gpu();
  for (auto& f : factors) set->add(f);
  lin.clear();
  for (auto& lf : set->calc_linear_factors(values)) lin.push_back(unpack(lf));
  set->error(values2);
  err.clear();
  for (auto& f : factors) err.push_back(f->error(values2));
}

int main(int argc, char** argv) {
  Case in(argc, argv);
  if (!in) return 2;
  const auto tp = in.next(), tc = in.next(), sp = in.next(), sc = in.next();  // N x 4 (x, y, z, 1), N x 16
  const auto Tt = in.next(), Ts = in.next(), Ts2 = in.next();
  const std::size_t nt = tp.size() / 4, ns = sp.size() / 4;

  auto target = std::make_shared<PointCloudGPU>(tp.data(), tc.data(), nt);
  auto source = std::make_shared<PointCloudGPU>(sp.data(), sc.data(), ns);
  auto voxels = std::make_shared<GaussianVoxelMapGPU>(0.5);
  voxels->insert(tp.data(), 4, tc.data(), 16, nt);

  // the reference's OffloadableGPU calls, through the base class
  std::vector<OffloadableGPU::Ptr> objects = {voxels, source, target};
  const std::uint64_t t0 = OffloadableGPU::current_access_time();
  for (auto& o : objects) {
    EXPECT(o->loaded_on_gpu() && o->memory_usage_gpu() > 0);
    const std::size_t bytes = o->memory_usage_gpu();
    EXPECT(o->offload_gpu() && !o->offload_gpu());
    EXPECT(!o->loaded_on_gpu() && o->memory_usage_gpu() == 0);
    EXPECT(o->reload_gpu() && !o->reload_gpu() && o->memory_usage_gpu() == bytes);
    EXPECT(o->offload_gpu() && o->touch() && o->loaded_on_gpu() && !o->touch());
  }
  EXPECT(OffloadableGPU::current_access_time() == t0 + 2 * objects.size());
  EXPECT(source->last_accessed_time() == t0 + 3);
  for (auto& o : objects) EXPECT(with_stream(o, nullptr));
  // a map with nothing inserted has no device map yet: it reports the clock's value at its construction and moves nothing
  const std::uint64_t t1 = OffloadableGPU::current_access_time();
  OffloadableGPU::Ptr unbuilt = std::make_shared<GaussianVoxelMapGPU>(0.5);
  EXPECT(unbuilt->last_accessed_time() == t1 && unbuilt->loaded_on_gpu() && unbuilt->memory_usage_gpu() == 0);
  EXPECT(!unbuilt->offload_gpu() && !unbuilt->reload_gpu());
  EXPECT(!unbuilt->touch() && unbuilt->last_accessed_time() == t1 && OffloadableGPU::current_access_time() == t1 + 1);

  Values values, values2;
  insert_pose(values, 0, Tt);
  insert_pose(values, 1, Ts);
  insert_pose(values2, 0, Tt);
  insert_pose(values2, 1, Ts2);

  auto vgicp = std::make_shared<IntegratedVGICPFactor>(Key(0), Key(1), voxels, source);
  auto tree = std::make_shared<KdTreeGPU>(target);
  auto gicp = std::make_shared<IntegratedGICPFactor>(Key(0), Key(1), target, source, tree);
  auto icp = std::make_shared<IntegratedICPFactor>(Key(0), Key(1), target, source, tree, false, nullptr);
  std::vector<Hess> lin0, lin1;
  std::vector<double> err0, err1;
  step({vgicp, gicp, icp}, values, values2, lin0, err0);
  EXPECT(lin0.size() == 3 && lin0[0].f > 0.0);

  // the same factors with offloading on, every object offloaded before each step: the launches reload what they read
  std::vector<std::shared_ptr<IntegratedMatchingCostFactorB200>> offloading = {vgicp, gicp, icp};
  for (auto& f : offloading) {
    f->set_enable_offloading(true);
    EXPECT(f->memory_usage_gpu() > 0);
  }
  for (int rep = 0; rep < 2; rep++) {
    for (auto& o : objects) o->offload_gpu();
    step(offloading, values, values2, lin1, err1);
    for (int i = 0; i < 3; i++) {
      EXPECT(same_hess(lin0[i], lin1[i]));
      EXPECT(std::memcmp(&err0[i], &err1[i], sizeof(double)) == 0);
    }
    EXPECT(voxels->loaded_on_gpu() && source->loaded_on_gpu());
    EXPECT(!target->loaded_on_gpu());  // the kd-tree factors read their own target records
  }
  // clone() carries the setting over
  auto copy = std::dynamic_pointer_cast<IntegratedMatchingCostFactorB200>(vgicp->clone());
  for (auto& o : objects) o->offload_gpu();
  step({copy}, values, values2, lin1, err1);
  EXPECT(same_hess(lin0[0], lin1[0]));
  // with offloading off, a factor that would read an offloaded object throws
  auto plain = std::make_shared<IntegratedVGICPFactor>(Key(0), Key(1), voxels, source);  // made while the objects are resident
  voxels->offload_gpu();
  bool threw = false;
  try {
    plain->error(values2);
  } catch (const std::exception&) {
    threw = true;
  }
  EXPECT(threw && !voxels->loaded_on_gpu());
  std::printf("OK\n");
  return 0;
}
