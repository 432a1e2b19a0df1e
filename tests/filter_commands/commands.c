/* tests/filter_commands/commands.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Linked with oracle/ff_driver.c and transform360_cuda: what avfilter_process_command does (sendcmd, zmq), and
 * av_opt_get_double on the filter's private context, for a filter the driver opened.
 */
#include "avfilter.h"

extern AVFilter ff_vf_transform360_cuda;

/* oracle/ff_driver.c's filter instance; its first member is the filter's AVFilterContext */
typedef struct T360Filter T360Filter;
static AVFilterContext* context_of(const T360Filter* f) { return (AVFilterContext*)f; }

__attribute__((visibility("default"))) int t360f_command(T360Filter* f, const char* cmd, const char* arg) {
  char res[256] = {0};
  if (!ff_vf_transform360_cuda.process_command) return AVERROR(ENOSYS);
  return ff_vf_transform360_cuda.process_command(context_of(f), cmd, arg, res, (int)sizeof(res), 0);
}

/* the current value of a numeric option; ENOENT for other names */
__attribute__((visibility("default"))) int t360f_option(const T360Filter* f, const char* name, double* value) {
  for (const AVOption* o = ff_vf_transform360_cuda.priv_class->option; o->name; o++) {
    if (o->type == AV_OPT_TYPE_CONST || strcmp(o->name, name)) continue;
    const uint8_t* src = (const uint8_t*)context_of(f)->priv + o->offset;
    if (o->type == AV_OPT_TYPE_FLOAT) *value = *(const float*)src;
    else if (o->type == AV_OPT_TYPE_INT) *value = *(const int*)src;
    else return AVERROR(ENOENT);
    return 0;
  }
  return AVERROR(ENOENT);
}
