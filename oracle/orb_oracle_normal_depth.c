/* orb_oracle_normal_depth.c -- CPU ORACLE (test infrastructure only; never linked into liborbfe.so) of
 * MapPoint::UpdateNormalAndDepth (src/MapPoint.cc:273-312) as OpenCV 2.4's cv::Mat algebra evaluates it (DESIGN.md §2):
 *   normali = mWorldPos - Owi                  float subtraction per component
 *   normal + normali/cv::norm(normali)         scaleAdd(normali, (float)(1.0/norm), normal): float product, then float add
 *   cv::norm                                   sqrt of the double sum of squares, x, y, z in order
 *   normal/n                                   convertTo scaling: normal_k * (float)(1.0/n) + 0.0f
 *   mfMinDistance = (1.0f/scaleFactor)*dist / GetScaleFactor(level), mfMaxDistance = scaleFactor*dist * GetScaleFactor(nLevels-1-level)
 * Host arrays in the layout of orbfe_normal_and_depth.  Built into oracle/liborb_oracle.so as its own object by
 * oracle/Makefile (-ffp-contract=off: no FMA); pinned to the reference's own
 * UpdateNormalAndDepth by tests/test_oracle_normal_depth.py.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

void orb_oracle_normal_depth(int npoints, const float *world, const float *ref_centers, const int32_t *ref_octave, const int32_t *group_ptr,
                             const float *obs_centers, float scale_factor, int nlevels, const float *scale_factors, float *normal_out,
                             float *min_dist_out, float *max_dist_out);

static double norm3(const float *v) { /* normL2_32f: double accumulation of v*v, then sqrt */
    double s = 0;
    for (int k = 0; k < 3; k++) s += (double)v[k] * (double)v[k];
    return sqrt(s);
}

/* Point g with an empty group is left untouched (MapPoint.cc:281-282, a bad point returns before writing). */
void orb_oracle_normal_depth(int npoints, const float *world, const float *ref_centers, const int32_t *ref_octave, const int32_t *group_ptr,
                             const float *obs_centers, float scale_factor, int nlevels, const float *scale_factors, float *normal_out,
                             float *min_dist_out, float *max_dist_out) {
    for (int g = 0; g < npoints; g++) {
        const int b = group_ptr[g], e = group_ptr[g + 1];
        if (e <= b) continue;
        const float *P = world + 3 * (size_t)g;
        float normal[3] = {0.0f, 0.0f, 0.0f};
        for (int j = b; j < e; j++) {
            float d[3];
            for (int k = 0; k < 3; k++) d[k] = P[k] - obs_centers[3 * (size_t)j + k];
            const float a = (float)(1.0 / norm3(d));
            for (int k = 0; k < 3; k++) normal[k] = d[k] * a + normal[k];
        }
        const float inv_n = (float)(1.0 / (double)(e - b));
        for (int k = 0; k < 3; k++) normal_out[3 * (size_t)g + k] = normal[k] * inv_n + 0.0f;
        float pc[3];
        for (int k = 0; k < 3; k++) pc[k] = P[k] - ref_centers[3 * (size_t)g + k];
        const float dist = (float)norm3(pc);
        const int level = ref_octave[g];
        min_dist_out[g] = (1.0f / scale_factor) * dist / scale_factors[level];
        max_dist_out[g] = scale_factor * dist * scale_factors[nlevels - 1 - level];
    }
}
