// oracle/_ref — the coloured scan of LIVMapper::publish_frame_world (src/LIVMapper.cpp:1140-1173) on the reference's OWN
// VIOManager::updateFrameState (src/vio.cpp:1690-1697), Frame::w2f / w2c (include/frame.h), vk::AbstractCamera::isInFrame (the
// vikit stand-in of ref_shim/) and VIOManager::getInterpolatedPixel (src/vio.cpp:1742-1760), on the VIOManager the driver
// ref_vio.cpp (included as it is) creates; PointXYZRGB is the stand-in of ref_shim/pcl. LIVMapper itself is bound to ROS and
// is not compiled: the per-point loop of publish_frame_world and RGBpointBodyToWorld (:682-690) are restated here, statement
// for statement. TEST INFRASTRUCTURE ONLY: pins the oracle's restatement (oracle/orc_color.cpp) in tests/test_oracle_color.py.
// Built by oracle/color.mk where the reference source exists.
#include "ref_vio.cpp"

extern "C" {

// RGBpointBodyToWorld with _state = the packed `state`, extR / extT of LIVMapper (lidar -> imu): world_out n x 3
void ref_color_world(const double *extR, const double *extT, const double *state, const float *pts, int n, float *world_out) {
  StatesGroup s;
  unpack_state(state, s);
  M3D R;
  V3D t(extT[0], extT[1], extT[2]);
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) R(a, b) = extR[3 * a + b];
  for (int i = 0; i < n; i++) {
    V3D p_body(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
    V3D p_global(s.rot_end * (R * p_body + t) + s.pos_end);
    world_out[3 * i] = p_global(0), world_out[3 * i + 1] = p_global(1), world_out[3 * i + 2] = p_global(2);
  }
}

// publish_frame_world's loop over the world cloud with img_rgb = `bgr` (CV_8UC3 of the camera's size) after
// updateFrameState(state); outputs as orc_color_colorize. Returns n_kept.
int ref_color_colorize(void *h, const float *cloud, int n, const uint8_t *bgr, const double *state, double blind_rgb_points, float *xyz_out, uint8_t *bgr_out,
                       int32_t *index_out) {
  RefVio *r = (RefVio *)h;
  VIOManager &v = r->v;
  StatesGroup s;
  unpack_state(state, s);
  cv::Mat grey(v.height, v.width, CV_8UC1);
  v.new_frame_.reset(new Frame(v.cam, grey));
  v.updateFrameState(s);
  cv::Mat img_rgb(v.height, v.width, CV_8UC3, (void *)bgr);
  int kept = 0;
  for (int i = 0; i < n; i++) {
    pcl::PointXYZRGB pointRGB;
    pointRGB.x = cloud[3 * i], pointRGB.y = cloud[3 * i + 1], pointRGB.z = cloud[3 * i + 2];
    V3D p_w(cloud[3 * i], cloud[3 * i + 1], cloud[3 * i + 2]);
    V3D pf(v.new_frame_->w2f(p_w));
    if (pf[2] < 0) continue;
    V2D pc(v.new_frame_->w2c(p_w));
    if (v.new_frame_->cam_->isInFrame(pc.cast<int>(), 3)) {
      V3F pixel = v.getInterpolatedPixel(img_rgb, pc);
      pointRGB.r = pixel[2];
      pointRGB.g = pixel[1];
      pointRGB.b = pixel[0];
      if (pf.norm() > blind_rgb_points) {
        xyz_out[3 * kept] = pointRGB.x, xyz_out[3 * kept + 1] = pointRGB.y, xyz_out[3 * kept + 2] = pointRGB.z;
        bgr_out[3 * kept] = pointRGB.b, bgr_out[3 * kept + 1] = pointRGB.g, bgr_out[3 * kept + 2] = pointRGB.r;
        index_out[kept++] = i;
      }
    }
  }
  return kept;
}
}
